"""Argument validation of the networks' fused tail kernels, without a GPU: every case here is refused
before any launch, so dummy host pointers stand in for the device tensors.  Each call must return
G6D_EINVAL with a message that names the offending argument."""
import ctypes as C

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


@pytest.fixture(scope='module')
def dummy():
    buf = (C.c_float * 16)()       # never dereferenced: validation fails first
    return C.c_void_p(C.addressof(buf)), buf


def _maps(n_scales, dummy, hs=33, ws=60, rfn=3, h0=(8, 16, 32, 64, 128, 256, 512, 1024)):
    m = _lib.DetMaps()
    m.n_scales, m.rfn, m.hs, m.ws = n_scales, rfn, hs, ws
    for s in range(min(n_scales, _lib.G6D_DET_MAX_SCALES)):
        for l in range(3):
            m.map[s][l] = dummy[0].value
            m.H[s][l], m.W[s][l] = h0[s] >> l, (2 * h0[s]) >> l
    m.mu[:] = [0.0, 0.0, 0.0]
    m.inv_sigma[:] = [1.0, 1.0, 1.0]
    m.clip = 10.0
    return m


def _fuse(lib, m, dummy, qn=1):
    p = dummy[0]
    return lib.g6d_det_score_fuse(C.byref(m), qn, p, p, p, p, p, None)


@pytest.mark.parametrize('s,l,dh,dw', [(0, 1, 1, 0), (2, 2, 0, -1), (3, 1, 0, 1), (1, 2, -1, 0)])
def test_det_score_fuse_rejects_inconsistent_level_sizes(lib, dummy, s, l, dh, dw):
    m = _maps(4, dummy)
    m.H[s][l] += dh
    m.W[s][l] += dw
    assert _fuse(lib, m, dummy) == G6D_EINVAL
    msg = lib.g6d_last_error()
    assert f'scale {s} level {l}'.encode() in msg, msg


def test_det_score_fuse_rejects_odd_level0(lib, dummy):
    """Level 0 of 15 rows: 15 >> 1 = 7 rows at level 1 would leave row 14 of the nearest x2 upsampling unmatched."""
    m = _maps(1, dummy)
    m.H[0][0], m.H[0][1], m.H[0][2] = 15, 7, 3
    assert _fuse(lib, m, dummy) == G6D_EINVAL
    assert b'scale 0 level 1' in lib.g6d_last_error()


@pytest.mark.parametrize('field', ['hs', 'ws', 'rfn'])
def test_det_score_fuse_rejects_empty_output(lib, dummy, field):
    m = _maps(2, dummy)
    setattr(m, field, 0)
    assert _fuse(lib, m, dummy) == G6D_EINVAL
    assert f'{field}=0'.encode() in lib.g6d_last_error()


@pytest.mark.parametrize('n_scales', [0, 7, 8])
def test_det_score_fuse_rejects_scale_count(lib, dummy, n_scales):
    m = _maps(n_scales, dummy)
    assert _fuse(lib, m, dummy) == G6D_EINVAL
    assert f'n_scales={n_scales}'.encode() in lib.g6d_last_error()


def test_det_score_fuse_rejects_null_map(lib, dummy):
    m = _maps(3, dummy)
    m.map[2][1] = None
    assert _fuse(lib, m, dummy) == G6D_EINVAL
    assert b'map[2][1] is null' in lib.g6d_last_error()


def _fill(lib, dummy, Q=1, R=6, fh=32, fw=32, Cc=128, sn=32, img_h=128, img_w=128):
    p = dummy[0]
    return lib.g6d_ref_volume_fill(p, p, p, p, p, p, Q, R, fh, fw, Cc, sn, img_h, img_w, p, p, None)


@pytest.mark.parametrize('kw,what', [(dict(R=1), b'2 <= R <= 7'), (dict(R=8), b'2 <= R <= 7'), (dict(Cc=6), b'C%4 == 0'),
                                     (dict(sn=1), b'sn >= 2'), (dict(R=0), b'2 <= R <= 7'), (dict(Cc=0), b'C%4 == 0')])
def test_ref_volume_fill_rejects_bad_dims(lib, dummy, kw, what):
    assert _fill(lib, dummy, **kw) == G6D_EINVAL
    msg = lib.g6d_last_error()
    assert b'g6d_ref_volume_fill' in msg and what in msg, msg
    (k, v), = kw.items()
    assert f'{"C" if k == "Cc" else k}={v} '.encode() in msg, msg
