"""Descriptor validation of the tensor-core convolution, without a GPU: every entry point (supported,
workspace_bytes, g6d_conv_tc) rejects a descriptor the kernels cannot run, whichever kernel its shape would
go to.  g6d_conv_tc is called with null tensor pointers, so nothing can launch: the descriptor error must be
reported before the pointer check."""
import ctypes

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(k):
    """64 -> 64 channels over one 32x32 image: k = 3 is a stride-1 3x3 (the A-reuse kernel), k = 1 a 1x1 (the
    persistent kernel)."""
    p = k // 2
    return _lib.ConvDesc(B=1, D=1, H=32, W=32, Cin=64, in_cstride=64, in_coff=0, Cout=64, kd=1, kh=k, kw=k, stride=1,
                         pd=0, ph=p, pw=p, Do=1, Ho=32, Wo=32, out_cstride=64, out_coff=0, prologue=0, group_rows=1,
                         act=0, max_chain_k=0)


BAD = {'out_slice': (dict(out_coff=8), b'output channel slice out of row'),
       'in_slice': (dict(in_coff=4), b'input channel slice out of row'),
       'prologue': (dict(prologue=9), b'bad prologue/act'),
       'act': (dict(act=7), b'bad prologue/act')}


def conv_tc(lib, d, kind):
    return lib.g6d_conv_tc(ctypes.byref(d), None, None, None, 64, kind, None, None, None, None, None, None, 0, None)


@pytest.mark.parametrize('kind', [_lib.TC_F16, _lib.TC_TF32])
@pytest.mark.parametrize('k', [3, 1])
def test_valid_descriptor_is_accepted(lib, k, kind):
    d = desc(k)
    assert lib.g6d_conv_tc_supported(ctypes.byref(d), kind) == 1
    assert lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), kind) >= 0
    assert conv_tc(lib, d, kind) == G6D_EINVAL
    assert b'null tensor pointer' in lib.g6d_last_error()


@pytest.mark.parametrize('bad', sorted(BAD))
@pytest.mark.parametrize('kind', [_lib.TC_F16, _lib.TC_TF32])
@pytest.mark.parametrize('k', [3, 1])
def test_bad_descriptor_is_rejected_everywhere(lib, k, kind, bad):
    fields, msg = BAD[bad]
    d = desc(k)
    for name, v in fields.items():
        setattr(d, name, v)
    assert lib.g6d_conv_tc_supported(ctypes.byref(d), kind) == 0
    assert lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), kind) == -1
    assert conv_tc(lib, d, kind) == G6D_EINVAL
    err = lib.g6d_last_error()
    assert msg in err, err
