"""g6d_conv_tc_plan_ex / g6d_conv_tc_workspace_bytes_ex without a GPU: G6D_TC_PRENORM puts prologue layers on the
split input exactly where a layer without a prologue would get it, adds the split copy to the workspace, and changes
nothing anywhere else; flags = 0 is the plain entry points; bad descriptors are rejected with the same messages."""
import ctypes

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(k=3, H=8, W=8, Cin=512, Cout=128, B=320, prologue=_lib.PRO_CORR, group_rows=320):
    p = k // 2
    return _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=Cin, in_cstride=Cin, in_coff=0, Cout=Cout, kd=1, kh=k, kw=k, stride=1,
                         pd=0, ph=p, pw=p, Do=1, Ho=H, Wo=W, out_cstride=Cout, out_coff=0, prologue=prologue,
                         group_rows=group_rows, act=0, max_chain_k=0)


def plan(lib, d, kind, flags):
    out = (ctypes.c_int * 4)(-7, -7, -7, -7)
    rc = lib.g6d_conv_tc_plan_ex(ctypes.byref(d), kind, flags, out)
    return rc, list(out)


def ws(lib, d, kind, flags):
    return lib.g6d_conv_tc_workspace_bytes_ex(ctypes.byref(d), kind, flags)


PROS = [_lib.PRO_CORR, _lib.PRO_AFFINE, _lib.PRO_AFFINE_RELU]


# the selector towers' persistent-kernel layers: level 1 / 2 first convolutions (K = 4608) and the later 8x8 / 4x4 ones
@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('shape', [dict(H=8, W=8, Cin=512, Cout=128), dict(H=4, W=4, Cin=512, Cout=256),
                                   dict(H=8, W=8, Cin=128, Cout=128), dict(H=4, W=4, Cin=256, Cout=256)])
def test_prenorm_plan_and_workspace(lib, pro, shape):
    d = desc(prologue=pro, **shape)
    rc, pre = plan(lib, d, _lib.TC_F16, _lib.TC_PRENORM)
    assert rc == 0
    rc, gather = plan(lib, d, _lib.TC_F16, 0)
    assert rc == 0
    assert pre[0] == 0 and pre[3] == 1                       # persistent kernel, A by TMA im2col
    assert gather[3] == 0 and pre[:3] == gather[:3]          # kernel, BN and K splits do not depend on the flag
    splits = pre[2]
    M = d.B * d.Ho * d.Wo
    partials = splits * M * d.Cout * 4 if splits > 1 else 0
    assert ws(lib, d, _lib.TC_F16, 0) == partials
    assert ws(lib, d, _lib.TC_F16, _lib.TC_PRENORM) == (partials + 255) // 256 * 256 + d.B * d.H * d.W * d.Cin * 4


def test_flags_zero_is_the_plain_entry_points(lib):
    for d in (desc(), desc(prologue=_lib.PRO_NONE), desc(k=1), desc(H=32, W=32, Cin=64, Cout=64, B=1)):
        for kind in (_lib.TC_F16, _lib.TC_TF32):
            out = (ctypes.c_int * 4)()
            assert lib.g6d_conv_tc_plan(ctypes.byref(d), kind, out) == 0
            assert plan(lib, d, kind, 0) == (0, list(out))
            assert ws(lib, d, kind, 0) == lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), kind)


def test_prenorm_without_prologue_changes_nothing(lib):
    d = desc(prologue=_lib.PRO_NONE)
    assert plan(lib, d, _lib.TC_F16, _lib.TC_PRENORM) == plan(lib, d, _lib.TC_F16, 0)
    assert plan(lib, d, _lib.TC_F16, 0)[1][3] == 1
    assert ws(lib, d, _lib.TC_F16, _lib.TC_PRENORM) == ws(lib, d, _lib.TC_F16, 0)


@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('why, fields, kind, kernel', [
    ('1x1', dict(kh=1, kw=1, ph=0, pw=0), _lib.TC_F16, 0),
    ('stride 2', dict(stride=2, Ho=4, Wo=4), _lib.TC_F16, 0),
    ('3-D', dict(D=3, kd=3, pd=1, Do=3), _lib.TC_F16, 0),
    ('tf32', {}, _lib.TC_TF32, 0),
    ('A-reuse', dict(H=32, W=32, Ho=32, Wo=32, B=2, group_rows=2), _lib.TC_F16, 1),
])
def test_prenorm_is_a_noop_elsewhere(lib, pro, why, fields, kind, kernel):
    d = desc(prologue=pro)
    for name, v in fields.items():
        setattr(d, name, v)
    rc, pre = plan(lib, d, kind, _lib.TC_PRENORM)
    assert rc == 0, why
    assert pre == plan(lib, d, kind, 0)[1], why
    assert pre[0] == kernel and pre[3] == 0, why
    assert ws(lib, d, kind, _lib.TC_PRENORM) == ws(lib, d, kind, 0), why


@pytest.mark.parametrize('flags', [0, _lib.TC_PRENORM])
def test_prenorm_rejects_bad_descriptors(lib, flags):
    d = desc()
    d.out_coff = 8
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'output channel slice out of row' in lib.g6d_last_error()
    assert ws(lib, d, _lib.TC_F16, flags) == -1
    d = desc(Cin=96)
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'Cin (96) must be a multiple of 64' in lib.g6d_last_error()
    d = desc()
    d.in_coff = 64
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'input channel slice out of row' in lib.g6d_last_error()
    assert lib.g6d_conv_tc_plan_ex(ctypes.byref(desc()), _lib.TC_F16, flags, None) == G6D_EINVAL
    assert b'null output' in lib.g6d_last_error()


def test_unknown_flags_rejected(lib):
    assert plan(lib, desc(), _lib.TC_F16, 2)[0] == G6D_EINVAL
    assert b'bad flags' in lib.g6d_last_error()
    assert ws(lib, desc(), _lib.TC_F16, 2) == -1
