"""Multi-peak detection (g6d_det_parse_peaks) through its host twin, without a GPU: the selection against the numpy
restatement in det_peaks_oracle.py, bit for bit on the decoded rows, indices, masks and counts, and the argument checks."""
import ctypes as C

import numpy as np
import pytest

from gen6d_b200 import _lib

from det_peaks_oracle import box_ious, det_peaks

G6D_EINVAL = -1
F32 = np.float32
_libm = C.CDLL('libm.so.6')
_libm.exp2f.restype, _libm.exp2f.argtypes = C.c_float, [C.c_float]


def exp2f(v):
    """libm's exp2f, which the host twin's decode calls."""
    return F32(_libm.exp2f(float(v)))


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def host_peaks(lib, scores, scales, offsets, max_inst=4, radius=1, nms_iou=0.3, box_size=128.0, min_score=-np.inf, pool=8):
    n, hs, ws = scores.shape
    det = np.full((max_inst, n, 4), np.nan, F32)
    idx = np.full((max_inst, n), -7, np.int64)
    valid = np.full((max_inst, n), -7, np.int32)
    count = np.full(n, -7, np.int32)
    rc = lib.g6d_det_parse_peaks_host(_ptr(scores), _ptr(scales), _ptr(offsets), n, hs, ws, pool, max_inst, radius, nms_iou, box_size,
                                      min_score, _ptr(det), _ptr(idx), _ptr(valid), _ptr(count))
    assert rc == 0, lib.g6d_last_error()
    return det, idx, valid, count


def _maps(n, hs, ws, seed, plateau=False):
    rng = np.random.RandomState(seed)
    sc = rng.randn(n, hs, ws).astype(F32)
    if plateau:
        sc = np.round(sc).astype(F32)
    scl = (rng.randn(n, hs, ws) * 0.5).astype(F32)
    off = (rng.rand(n, hs, ws, 2) - 0.5).astype(F32)
    return np.ascontiguousarray(sc), np.ascontiguousarray(scl), np.ascontiguousarray(off)


def _check(lib, sc, scl, off, **kw):
    got = host_peaks(lib, sc, scl, off, **kw)
    want = det_peaks(sc, scl, off, pool_ratio=kw.pop('pool', 8), exp2=exp2f, **kw)
    det, idx, valid, count = got
    np.testing.assert_array_equal(idx, want[1])
    np.testing.assert_array_equal(valid, want[2])
    np.testing.assert_array_equal(count, want[3])
    assert det.tobytes() == want[0].tobytes()
    # row 0 is the argmax; valid rows form a prefix of length count; rows past it repeat row 0
    for j in range(sc.shape[0]):
        assert (valid[:count[j], j] == 1).all() and (valid[count[j]:, j] == 0).all()
        kept = max(int(count[j]), 1)
        for m in range(kept, det.shape[0]):
            assert det[m, j].tobytes() == det[0, j].tobytes() and idx[m, j] == idx[0, j]
    return got


@pytest.mark.parametrize('shape', [(1, 1), (2, 3), (9, 13), (30, 40), (135, 240)])
@pytest.mark.parametrize('box_size', [16.0, 128.0])
def test_random_maps(lib, shape, box_size):
    n = 1 if shape == (135, 240) else 3
    sc, scl, off = _maps(n, *shape, seed=shape[0] * 1000 + shape[1])
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=8, radius=1, nms_iou=0.3, box_size=box_size)
    if shape[0] * shape[1] > 100 and box_size == 16.0:
        assert (count > 1).all()              # small boxes: several instances survive


@pytest.mark.parametrize('radius', [0, 1, 2, 3])
def test_radius(lib, radius):
    sc, scl, off = _maps(2, 20, 25, seed=50 + radius)
    _check(lib, sc, scl, off, max_inst=16, radius=radius, nms_iou=0.5, box_size=8.0)


def test_plateaus(lib):
    sc, scl, off = _maps(3, 24, 31, seed=3, plateau=True)
    sc[2] = 1.0                               # one flat map: the argmax is cell 0 and no other cell is a peak
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=6, radius=1, nms_iou=0.2, box_size=8.0)
    assert idx[0, 2] == 0 and count[2] == 1
    _check(lib, sc, scl, off, max_inst=6, radius=0, nms_iou=0.2, box_size=8.0)


def test_nan_cells(lib):
    sc, scl, off = _maps(3, 16, 18, seed=4)
    sc[0, 3, 4] = np.nan                      # NaN at the argmax: instance 0 is invalid, the map reports no instance
    sc[1, 5, 5] = np.nan                      # NaN elsewhere: it is the argmax too
    sc[1, 10, 10] = np.nan
    sc[2, ::3, ::4] = np.nan
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=5, radius=1, nms_iou=0.3, box_size=8.0)
    assert idx[0, 0] == 3 * 18 + 4 and idx[0, 1] == 5 * 18 + 5
    assert (count == 0).all() and (valid == 0).all()
    # a NaN beats every cell of its window, so no cell next to it is a peak
    sc[0, 3, 4] = 0.0
    _check(lib, sc, scl, off, max_inst=5, radius=1, nms_iou=0.3, box_size=8.0)
    sc[:, :, :] = np.where(np.isnan(sc), F32(-np.inf), sc)
    sc[0, 0, 0] = np.nan                      # a NaN scale / offset only affects that cell's box
    scl[1, 2, 2] = np.nan
    off[2, 7, 7, 0] = np.nan
    _check(lib, sc, scl, off, max_inst=5, radius=1, nms_iou=0.3, box_size=8.0)


def test_all_minus_inf(lib):
    sc, scl, off = _maps(2, 7, 9, seed=5)
    sc[:] = -np.inf
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1)
    assert (idx[0] == 0).all() and (count == 1).all()         # -inf >= -inf: the argmax is valid without a threshold
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=0, box_size=1.0)
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1, min_score=-1e30)
    assert (count == 0).all()


def test_min_score_above_every_score(lib):
    sc, scl, off = _maps(3, 12, 12, seed=6)
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1, min_score=float(sc.max()) + 1)
    assert (count == 0).all() and (valid == 0).all()
    flat = sc.reshape(3, -1)
    np.testing.assert_array_equal(idx[0], flat.argmax(1))
    np.testing.assert_array_equal(det[0, :, 3], flat.max(1))
    # a threshold between the instances keeps a prefix
    _check(lib, sc, scl, off, max_inst=8, radius=1, box_size=8.0, min_score=1.0)


def test_more_instances_than_peaks(lib):
    sc, scl, off = _maps(2, 4, 4, seed=7)
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=16, radius=3, box_size=1.0)
    assert (count == 1).all()                 # a 4x4 map under radius 3 has exactly one peak
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=16, radius=0, box_size=1.0, nms_iou=1.0)
    assert (count == 16).all()
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=16, radius=1, box_size=1.0)
    assert (count < 16).all()


def _chain_maps():
    """Three peaks on a row, A > B > C, spaced so that A's box overlaps B's beyond the threshold, B's overlaps C's, and A's
    overlaps C's below it: B is suppressed by A, and C survives because B was never kept."""
    sc = np.full((1, 5, 40), -5.0, F32)
    scl = np.zeros((1, 5, 40), F32)           # scale 1: boxes of side box_size
    off = np.zeros((1, 5, 40, 2), F32)
    for x, v in ((5, 3.0), (9, 2.0), (13, 1.0)):
        sc[0, 2, x] = v
    return sc, scl, off


def test_suppression_chain(lib):
    sc, scl, off = _chain_maps()
    # box side 48 px, centres 32 px apart: IoU(A,B) = 16/80 = 0.2, IoU(A,C) = 0
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1, nms_iou=0.1, box_size=48.0, min_score=0.0)
    assert count[0] == 2 and idx[0, 0] == 2 * 40 + 5 and idx[1, 0] == 2 * 40 + 13
    ious = box_ious(sc, scl, off, box_size=48.0, exp2=exp2f, cells=[[85, 89, 93]])[0]
    assert ious[0, 1] > F32(0.1) and ious[1, 2] > F32(0.1) and not ious[0, 2] > F32(0.1)


def test_iou_equal_to_threshold_is_kept(lib):
    sc, scl, off = _chain_maps()
    iou_ab = box_ious(sc, scl, off, box_size=48.0, exp2=exp2f, cells=[[85, 89]])[0][0, 1]
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1, nms_iou=float(iou_ab), box_size=48.0, min_score=0.0)
    assert count[0] == 3 and list(idx[:3, 0]) == [85, 89, 93]
    below = float(np.nextafter(iou_ab, F32(0)))
    det, idx, valid, count = _check(lib, sc, scl, off, max_inst=4, radius=1, nms_iou=below, box_size=48.0, min_score=0.0)
    assert count[0] == 2 and list(idx[:2, 0]) == [85, 93]


def test_argument_errors(lib):
    sc, scl, off = _maps(2, 6, 6, seed=8)
    good = dict(max_inst=4, radius=1, nms_iou=0.3, box_size=128.0, min_score=-np.inf)
    bad = [dict(max_inst=0), dict(max_inst=_lib.G6D_DET_MAX_INSTANCES + 1), dict(radius=-1),
           dict(radius=_lib.G6D_DET_MAX_PEAK_RADIUS + 1), dict(nms_iou=-0.01), dict(nms_iou=1.01), dict(nms_iou=float('nan')),
           dict(box_size=0.0), dict(box_size=float('inf')), dict(min_score=float('nan'))]
    n, hs, ws = sc.shape
    out = [np.zeros((16, n, 4), F32), np.zeros((16, n), np.int64), np.zeros((16, n), np.int32), np.zeros(n, np.int32)]
    for b in bad:
        a = {**good, **b}
        rc = lib.g6d_det_parse_peaks_host(_ptr(sc), _ptr(scl), _ptr(off), n, hs, ws, 8, a['max_inst'], a['radius'], a['nms_iou'],
                                          a['box_size'], a['min_score'], *map(_ptr, out))
        assert rc == G6D_EINVAL, b
        assert b'g6d_det_parse_peaks_host' in lib.g6d_last_error()
    for shape in ((0, hs, ws, 8), (n, 0, ws, 8), (n, hs, -1, 8), (n, hs, ws, 0)):
        rc = lib.g6d_det_parse_peaks_host(_ptr(sc), _ptr(scl), _ptr(off), *shape, 4, 1, 0.3, 128.0, -np.inf, *map(_ptr, out))
        assert rc == G6D_EINVAL, shape
    rc = lib.g6d_det_parse_peaks_host(None, _ptr(scl), _ptr(off), n, hs, ws, 8, 4, 1, 0.3, 128.0, -np.inf, *map(_ptr, out))
    assert rc == G6D_EINVAL
    # the device entry point checks the same arguments before any launch (no device memory is touched)
    rc = lib.g6d_det_parse_peaks(_ptr(sc), _ptr(scl), _ptr(off), n, hs, ws, 8, 0, 1, 0.3, 128.0, -np.inf, *map(_ptr, out), None)
    assert rc == G6D_EINVAL and b'g6d_det_parse_peaks' in lib.g6d_last_error()
