"""Argument validation of the selector's streaming kernels and the shared layout / resize / normalisation
kernels, without a GPU: every case here is refused before any launch, so dummy host pointers stand in for
the device tensors.  Each call must return G6D_EINVAL with a message that names the entry point."""
import ctypes as C

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


_BUF = (C.c_float * 16)()         # never dereferenced: validation fails first


@pytest.fixture(scope='module')
def p():
    return C.c_void_p(C.addressof(_BUF))


def refused(lib, rc, *what):
    assert rc == G6D_EINVAL, rc
    msg = lib.g6d_last_error()
    for w in what:
        assert w in msg, msg


@pytest.mark.parametrize('Cc', [64, 127, 384, 1024, 0])
def test_sel_corr_score_rejects_channel_count(lib, p, Cc):
    refused(lib, lib.g6d_sel_corr_score(p, p, 4, 16, Cc, p, None), b'g6d_sel_corr_score', b'C must be 128, 256 or 512')


def test_sel_corr_score_rejects_too_many_locations(lib, p):
    """P scores of a slice live in dynamic shared memory: 8192 floats is the limit."""
    refused(lib, lib.g6d_sel_corr_score(p, p, 4, 8193, 512, p, None), b'g6d_sel_corr_score', b'P too large')


@pytest.mark.parametrize('n,Cc,heads', [(2049, 512, 8), (4096, 64, 1), (64, 512, 4), (64, 500, 8), (64, 0, 0)])
def test_attention_headmajor_rejects_bad_shapes(lib, p, n, Cc, heads):
    refused(lib, lib.g6d_attention_headmajor(p, p, p, p, n, Cc, heads, None), b'g6d_attention_headmajor',
            b'n <= 2048, C = heads * 64')


@pytest.mark.parametrize('n,Cc,heads', [(8192, 4096, 1), (12000, 512, 1), (1, 12288, 1), (8192, 8192, 2)])
def test_attention_rejects_shared_memory_overflow(lib, p, n, Cc, heads):
    """n + C/heads floats of dynamic shared memory plus the 32-float reduction buffer must fit in 48 KB; n = 8192
    with one head of 4096 channels is 48 KB of dynamic memory alone and would fail at launch."""
    assert n + Cc // heads > _lib.G6D_ATTENTION_MAX_SMEM_FLOATS
    rc = lib.g6d_attention(p, p, p, p, n, Cc, heads, None)
    refused(lib, rc, b'g6d_attention')
    if n <= 8192:
        assert b'shared memory' in lib.g6d_last_error()


def test_attention_shared_memory_bound_is_48k():
    assert 4 * (_lib.G6D_ATTENTION_MAX_SMEM_FLOATS + 32) == 48 * 1024


@pytest.mark.parametrize('Cc', [2, 6, 63, 514])
def test_maxpool_and_l2norm_reject_channels_not_multiple_of_4(lib, p, Cc):
    refused(lib, lib.g6d_maxpool2x2(p, p, 1, 4, 4, Cc, None), b'g6d_maxpool2x2', b'C%4==0')
    refused(lib, lib.g6d_l2norm_channels(p, p, 4, Cc, 1e-12, None), b'g6d_l2norm_channels')


@pytest.mark.parametrize('Cc,ics,ico,ocs,oco', [(6, 8, 0, 8, 0), (4, 10, 0, 8, 0), (4, 8, 2, 8, 0), (4, 8, 0, 6, 0),
                                                (4, 8, 0, 8, 1)])
def test_affine_act_rejects_unaligned_channels(lib, p, Cc, ics, ico, ocs, oco):
    """float4 loads and stores: every channel count, stride and offset is a multiple of 4."""
    refused(lib, lib.g6d_affine_act(p, p, 8, Cc, 8, p, p, 0, ics, ico, ocs, oco, None), b'g6d_affine_act', b'multiples of 4')


@pytest.mark.parametrize('fn', ['g6d_instnorm_stats', 'g6d_instnorm_partial'])
@pytest.mark.parametrize('rows,rpg,what', [(10, 3, b'bad args'), (100, 7, b'bad args'), (65536, 1, b'too many groups'),
                                           (2 * 65536, 2, b'too many groups')])
def test_instnorm_rejects_ragged_groups_and_group_count(lib, p, fn, rows, rpg, what):
    """rows must be whole groups, and groups ride on grid.y (<= 65535)."""
    if fn == 'g6d_instnorm_stats':
        rc = lib.g6d_instnorm_stats(p, rows, 4, 4, 0, rpg, 1e-5, p, p, p, None)
    else:
        rc = lib.g6d_instnorm_partial(p, rows, 4, 4, 0, rpg, p, None)
    refused(lib, rc, fn.encode(), what)


@pytest.mark.parametrize('fn', ['g6d_instnorm_stats', 'g6d_instnorm_partial'])
def test_instnorm_rejects_channels_past_the_row(lib, p, fn):
    if fn == 'g6d_instnorm_stats':
        rc = lib.g6d_instnorm_stats(p, 8, 64, 64, 4, 8, 1e-5, p, p, p, None)
    else:
        rc = lib.g6d_instnorm_partial(p, 8, 64, 64, 4, 8, p, None)
    refused(lib, rc, fn.encode())


@pytest.mark.parametrize('Cc,ocs,oco', [(8, 8, 1), (8, 16, 9), (8, 4, 0), (4, 100, 97)])
def test_resize_bilinear_rejects_channels_past_the_output_row(lib, p, Cc, ocs, oco):
    refused(lib, lib.g6d_resize_bilinear(p, p, 1, 4, 4, 8, 8, Cc, ocs, oco, None), b'g6d_resize_bilinear')
