"""One im2col A box per row of taps (x reuse) against the A-reuse kernel the same layers take without
G6D_TC_REUSE_IM2COL.  A BN 64 layer in that kernel's K order loads one box per (channel block, kz, ky) group over the
padded enumeration of Wo + kw - 1 columns and reads tap kx through a descriptor shifted by kx rows; every real output
element sums the same products in the same order, so outputs must be equal bit for bit.  The shapes put tile edges
across rows, planes and images, use the 1x15 correlation's row of taps, a small volume, folded and unfolded K splits,
and an output slice of a wider row whose other bytes must stay untouched."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


@pytest.fixture(autouse=True)
def f16(monkeypatch):
    monkeypatch.setenv('G6D_CONV_KIND', 'f16')
    monkeypatch.delenv('G6D_CONV_PATH', raising=False)


def plan6(x, pc, flags, out_cs=None):
    from gen6d_b200 import _lib
    if x.dim() == 4:
        B, H, W, cs = x.shape
        D = 1
    else:
        B, D, H, W, cs = x.shape
    kd, kh, kw = pc.k
    pd, ph, pw = pc.pad
    d = _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=0, Cout=pc.cout, kd=kd, kh=kh, kw=kw,
                      stride=1, pd=pd, ph=ph, pw=pw, Do=D + 2 * pd - kd + 1, Ho=H + 2 * ph - kh + 1,
                      Wo=W + 2 * pw - kw + 1, out_cstride=out_cs or pc.cout, out_coff=0, prologue=0, group_rows=1, act=0,
                      max_chain_k=pc.max_chain_k)
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_v2(ctypes.byref(d), pc.kind, flags, out, 6), 'g6d_conv_tc_plan_v2')
    return list(out)


def debug_clear():
    from gen6d_b200 import _lib
    rec = (ctypes.c_int * 8)()
    _lib.check(_lib.lib().g6d_conv_tc_debug(rec), 'g6d_conv_tc_debug')
    return list(rec)


def make(ops, shape, cout, k, pad, seed):
    gen = torch.Generator(device='cpu').manual_seed(seed)
    cin = shape[-1]
    x = torch.randn(*shape, generator=gen).cuda()
    w = torch.randn(cout, cin, *k, generator=gen) * (2 / (np.prod(k) * cin)) ** .5
    return x, ops.pack_conv(w.cuda(), torch.randn(cout, generator=gen).cuda(), pad=pad)


def run_both(ops, x, pc, flags, **kw):
    """(x reuse, A-reuse kernel) outputs; asserts the plans and a clean debug record after each call."""
    from gen6d_b200 import _lib
    xr, ref = plan6(x, pc, _lib.TC_REUSE_IM2COL | flags), plan6(x, pc, 0)
    assert xr[0] == 0 and xr[3] == 1 and xr[5] == 1 and xr[1] == 64
    assert ref[0] == 1 and ref[5] == 0
    assert xr[2] == ref[2]
    assert debug_clear()[0] == 0
    a = ops.conv(x, pc, reuse_im2col=True, fold_splits=bool(flags & _lib.TC_FOLD_SPLITS), act=ops.ACT_RELU, **kw)
    assert debug_clear()[0] == 0
    b = ops.conv(x, pc, act=ops.ACT_RELU, **kw)
    assert debug_clear()[0] == 0
    return a, b, xr


# (input shape, kernel, pad): tiles of the padded enumeration cross rows, planes and images, with a partial last tile
SHAPES = [
    ((3, 13, 13, 64), (3, 3), 1),             # Ho * Wp = 195: tiles span planes and images
    ((2, 7, 45, 128), (1, 15), (0, 7)),      # the correlation's row of 15 taps, Wp = 59
    ((2, 12, 40, 64), (1, 7), (0, 3)),
    ((1, 32, 32, 32, 64), (3, 3, 3), 1),     # the refiner's 32^3 volume
    ((3, 6, 10, 10, 128), (3, 3, 3), 1),     # a small volume: tiles span z-planes and volumes
]


@pytest.mark.parametrize('shape, k, pad', SHAPES)
def test_xreuse_bit_identical(ops, shape, k, pad):
    x, pc = make(ops, shape, 64, k, pad, seed=sum(shape))
    a, b, _ = run_both(ops, x, pc, 0)
    assert torch.equal(a, b)
    assert float(a.abs().max()) > 0


def test_xreuse_unfolded_splits(ops):
    """K splits over channel blocks through fp32 partials (tc.M rows, real rows only) and the reduce kernel."""
    x, pc = make(ops, (1, 6, 10, 10, 512), 64, (3, 3, 3), 1, seed=3)
    a, b, xr = run_both(ops, x, pc, 0)
    assert xr[2] > 1 and xr[4] == 0
    assert torch.equal(a, b)


def test_xreuse_folded_splits(ops):
    """The same splits summed inside the CTA (G6D_TC_FOLD_SPLITS) over the padded tiles."""
    from gen6d_b200 import _lib
    x, pc = make(ops, (66, 16, 16, 256), 64, (3, 3), 1, seed=5)
    pc.max_chain_k = 384
    a, b, xr = run_both(ops, x, pc, _lib.TC_FOLD_SPLITS)
    assert xr[2] > 1 and xr[4] == 1
    assert torch.equal(a, b)


def test_xreuse_moments(ops):
    """Fused InstanceNorm moments per plane: taken from y, within the fp64 reordering tolerance."""
    x, pc = make(ops, (2, 16, 16, 16, 64), 64, (3, 3, 3), 1, seed=9)
    (a, sa), (b, sb), _ = run_both(ops, x, pc, 0, stats_rows=16 ** 3)
    assert torch.equal(a, b)
    np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)


def test_xreuse_output_slice_untouched(ops):
    """Output channels [40, 104) of 136-wide rows over a NaN-filled buffer: padded rows are never written, nor is any
    byte outside the real outputs."""
    x, pc = make(ops, (3, 13, 13, 64), 64, (3, 3), 1, seed=13)
    out_a = torch.full((3, 13, 13, 136), float('nan'), device='cuda')
    out_b = out_a.clone()
    a, b, _ = run_both(ops, x, pc, 0)
    from gen6d_b200 import _lib
    assert plan6(x, pc, _lib.TC_REUSE_IM2COL, out_cs=136)[5] == 1
    ops.conv(x, pc, reuse_im2col=True, act=ops.ACT_RELU, out=out_a, out_coff=40)
    assert debug_clear()[0] == 0
    ops.conv(x, pc, act=ops.ACT_RELU, out=out_b, out_coff=40)
    torch.cuda.synchronize()
    assert torch.equal(out_a[..., 40:104], a)
    assert torch.equal(out_a[..., 40:104], out_b[..., 40:104])
    assert bool(torch.isnan(out_a[..., :40]).all()) and bool(torch.isnan(out_a[..., 104:]).all())
