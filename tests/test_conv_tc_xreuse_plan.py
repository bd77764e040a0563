"""g6d_conv_tc_plan_v2's sixth field without a GPU: one im2col A box per row of taps (x reuse) is planned for BN 64
layers in the A-reuse kernel's K order (G6D_TC_REUSE_IM2COL on a layer that kernel would take) with kw > 1, and for
nothing else; it changes neither the other plan fields nor the workspace."""
import ctypes

import pytest

from gen6d_b200 import _lib

RO = _lib.TC_REUSE_IM2COL | _lib.TC_PRENORM
F16 = _lib.TC_F16


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(B, D, H, W, Cin, Cout, k, pad, prologue=_lib.PRO_NONE):
    kd, kh, kw = k
    pd, ph, pw = pad
    return _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=Cin, in_cstride=Cin, in_coff=0, Cout=Cout, kd=kd, kh=kh, kw=kw, stride=1,
                         pd=pd, ph=ph, pw=pw, Do=D + 2 * pd - kd + 1, Ho=H + 2 * ph - kh + 1, Wo=W + 2 * pw - kw + 1,
                         out_cstride=Cout, out_coff=0, prologue=prologue, group_rows=1, act=0, max_chain_k=0)


def plan(lib, d, flags, n=6):
    out = (ctypes.c_int * 6)(*([-7] * 6))
    assert lib.g6d_conv_tc_plan_v2(ctypes.byref(d), F16, flags, out, n) == 0
    return list(out)


def ws(lib, d, flags):
    return lib.g6d_conv_tc_workspace_bytes_ex(ctypes.byref(d), F16, flags)


# bench.py's BN 64 layers in the A-reuse K order: the refiner's 32^3 volume net (10 poses), its 32^2 feature branches
# (70 crops) and the selector's 16x16 level-0 tower (320 reference x query pairs)
XR = [desc(10, 32, 32, 32, 256, 64, (3, 3, 3), (1, 1, 1)), desc(10, 32, 32, 32, 128, 64, (3, 3, 3), (1, 1, 1)),
      desc(10, 32, 32, 32, 64, 64, (3, 3, 3), (1, 1, 1), _lib.PRO_AFFINE_RELU),
      desc(70, 1, 32, 32, 256, 64, (1, 3, 3), (0, 1, 1)), desc(70, 1, 16, 16, 256, 64, (1, 3, 3), (0, 1, 1), _lib.PRO_AFFINE_RELU),
      desc(320, 1, 16, 16, 512, 64, (1, 3, 3), (0, 1, 1), _lib.PRO_AFFINE)]
# not x reuse: BN 128 and 32, the default K order (no flag), 1x1, kw = 1
NOT = [desc(10, 32, 32, 32, 128, 128, (3, 3, 3), (1, 1, 1)), desc(70, 1, 32, 32, 256, 256, (1, 3, 3), (0, 1, 1)),
       desc(10, 1, 88, 116, 256, 480, (1, 1, 15), (0, 0, 7)), desc(70, 1, 32, 32, 64, 32, (1, 3, 3), (0, 1, 1)),
       desc(70, 1, 32, 32, 256, 64, (1, 1, 1), (0, 0, 0)), desc(70, 1, 32, 32, 256, 64, (1, 3, 1), (0, 1, 0))]


@pytest.mark.parametrize('i', range(len(XR)))
def test_xreuse_planned(lib, i):
    d = XR[i]
    p = plan(lib, d, RO)
    assert p[0] == 0 and p[1] == 64 and p[3] == 1 and p[5] == 1
    assert plan(lib, d, 0)[5] == 0                        # flag-less: the A-reuse kernel, as before
    assert plan(lib, d, RO | _lib.TC_FOLD_SPLITS)[5] == 1


@pytest.mark.parametrize('i', range(len(NOT)))
def test_xreuse_not_planned(lib, i):
    for flags in (0, RO, RO | _lib.TC_FOLD_SPLITS):
        assert plan(lib, NOT[i], flags)[5] == 0


@pytest.mark.parametrize('i', range(len(XR)))
def test_xreuse_workspace_and_fields_unchanged(lib, i):
    """The workspace is the split-K partials of the real rows (none when folded) followed by the split input."""
    d = XR[i]
    for flags in (RO, RO | _lib.TC_FOLD_SPLITS):
        p = plan(lib, d, flags)
        M = d.B * d.Do * d.Ho * d.Wo
        partials = p[2] * M * d.Cout * 4 if p[2] > 1 and not p[4] else 0
        assert ws(lib, d, flags) == (partials + 255) // 256 * 256 + d.B * d.D * d.H * d.W * d.Cin * 4


def test_plan_v2_writes_n_fields(lib):
    p = plan(lib, XR[0], RO, n=5)
    assert p[5] == -7 and p[3] == 1
