"""Argument checks of g6d_det_corr_rowsum_objects, without a GPU: with null tensor pointers or a bad shape the entry
point must return G6D_EINVAL with its message before anything could launch."""
import ctypes

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1
MSG = b'g6d_det_corr_rowsum_objects: bad args'


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


BUF = ctypes.c_void_p(16)       # never dereferenced: every call below is rejected before a launch

# (partial, out, n_obj, qn, H, W, k, rfn)
GOOD = (BUF, BUF, 3, 2, 11, 13, 15, 32)
BAD = {'null_partial': dict(partial=None), 'null_out': dict(out=None), 'rfn_not_multiple_of_4': dict(rfn=30),
       'rfn_zero': dict(rfn=0), 'n_obj_zero': dict(n_obj=0), 'n_obj_negative': dict(n_obj=-2), 'k_zero': dict(k=0),
       'k_negative': dict(k=-1), 'qn_zero': dict(qn=0), 'H_zero': dict(H=0), 'W_zero': dict(W=0)}
FIELDS = ('partial', 'out', 'n_obj', 'qn', 'H', 'W', 'k', 'rfn')


@pytest.mark.parametrize('bad', sorted(BAD))
def test_bad_arguments_are_rejected(lib, bad):
    args = dict(zip(FIELDS, GOOD))
    args.update(BAD[bad])
    before = lib.g6d_launch_count()
    rc = lib.g6d_det_corr_rowsum_objects(*[args[f] for f in FIELDS], None)
    assert rc == G6D_EINVAL
    assert MSG in lib.g6d_last_error()
    assert lib.g6d_launch_count() == before


def test_entry_point_is_declared_and_bound():
    assert 'g6d_det_corr_rowsum_objects' in _lib.header_symbols()
    assert 'g6d_det_corr_rowsum_objects' in _lib._SIGNATURES
