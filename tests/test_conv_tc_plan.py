"""g6d_conv_tc_plan without a GPU: it reports the kernel, BN and K splits g6d_conv_tc would launch, agrees with
g6d_conv_tc_workspace_bytes on the splits, and rejects what the other entry points reject, with their message."""
import ctypes

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(k, H=32, W=32, Cin=64, Cout=64, B=1):
    p = k // 2
    return _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=Cin, in_cstride=Cin, in_coff=0, Cout=Cout, kd=1, kh=k, kw=k, stride=1,
                         pd=0, ph=p, pw=p, Do=1, Ho=H, Wo=W, out_cstride=Cout, out_coff=0, prologue=0, group_rows=1,
                         act=0, max_chain_k=0)


def plan(lib, d, kind):
    out = (ctypes.c_int * 4)(-7, -7, -7, -7)
    rc = lib.g6d_conv_tc_plan(ctypes.byref(d), kind, out)
    return rc, list(out)


@pytest.mark.parametrize('kind', [_lib.TC_F16, _lib.TC_TF32])
@pytest.mark.parametrize('case, kernel, bn', [
    (dict(k=3), 1, 64),                                   # 3x3 over a 32-wide plane: the A-reuse kernel
    (dict(k=1), 0, 64),                                   # 1x1: nothing to reuse, the persistent kernel
    (dict(k=3, H=120, W=160, Cout=256, B=10), 0, 128),    # halo too wide for shared memory: persistent
    (dict(k=3, Cout=32), 1, 32),
])
def test_plan_reports_kernel_bn_and_splits(lib, kind, case, kernel, bn):
    d = desc(**case)
    rc, (k, b, splits, split_in) = plan(lib, d, kind)
    assert rc == 0
    assert (k, b) == (kernel, bn)
    assert splits >= 1
    # the split input: only the persistent kernel, fp16, multi-tap
    assert split_in == int(kernel == 0 and kind == _lib.TC_F16 and d.kh > 1)
    ws = lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), kind)
    M = d.B * d.Do * d.Ho * d.Wo
    partials = splits * M * d.Cout * 4 if splits > 1 else 0
    split_bytes = d.B * d.H * d.W * d.Cin * 4
    assert ws == ((partials + 255) // 256 * 256 + split_bytes if split_in else partials)


BIG = dict(k=3, H=120, W=160, Cout=256, B=10)            # a persistent-kernel 3x3


@pytest.mark.parametrize('why, fields, kind', [
    ('tf32', {}, _lib.TC_TF32),
    ('prologue', dict(prologue=_lib.PRO_AFFINE), _lib.TC_F16),
    ('stride 2', dict(stride=2, Ho=60, Wo=80), _lib.TC_F16),
    ('3-D', dict(D=3, kd=3, pd=1, Do=3), _lib.TC_F16),
])
def test_split_input_only_where_it_applies(lib, why, fields, kind):
    d = desc(**BIG)
    for name, v in fields.items():
        setattr(d, name, v)
    rc, (k, _, _, split_in) = plan(lib, d, kind)
    assert rc == 0 and k == 0, why
    assert split_in == 0, why


@pytest.mark.parametrize('bad, fields', [('Cin % 64', dict(Cin=96, in_cstride=96)),
                                         ('input slice out of row', dict(in_coff=64))])
def test_split_input_descriptor_rejected(lib, bad, fields):
    d = desc(**BIG)
    for name, v in fields.items():
        setattr(d, name, v)
    assert plan(lib, d, _lib.TC_F16)[0] == G6D_EINVAL, bad
    assert lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), _lib.TC_F16) == -1


@pytest.mark.parametrize('kind', [_lib.TC_F16, _lib.TC_TF32])
def test_plan_rejects_bad_descriptors(lib, kind):
    d = desc(3)
    d.out_coff = 8
    assert plan(lib, d, kind)[0] == G6D_EINVAL
    assert b'output channel slice out of row' in lib.g6d_last_error()
    assert lib.g6d_conv_tc_plan(ctypes.byref(desc(3)), kind, None) == G6D_EINVAL
    assert b'null output' in lib.g6d_last_error()
