"""Prologue layers on the persistent kernel's split input (G6D_TC_PRENORM: the split pass applies the folded
InstanceNorm(+ReLU) or correlation prologue, then the kernel loads A by TMA im2col) against the producer warps, which
gather and transform the input once per tap.  The tiles are the same bytes by construction, so outputs must be equal
bit for bit, and the fused moments up to the order of their fp64 atomic additions."""
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


def plan(x, pc, prologue, group_rows, flags, in_coff=0):
    from gen6d_b200 import _lib
    B, H, W, cs = x.shape
    d = _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=in_coff, Cout=pc.cout, kd=1, kh=3, kw=3,
                      stride=1, pd=0, ph=1, pw=1, Do=1, Ho=H, Wo=W, out_cstride=pc.cout, out_coff=0, prologue=prologue,
                      group_rows=group_rows, act=0, max_chain_k=0)
    out = (ctypes.c_int * 4)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_ex(ctypes.byref(d), pc.kind, flags, out), 'g6d_conv_tc_plan_ex')
    return list(out)


def layer(ops, B, H, W, cin, cout, pro, group_rows, seed, cs=None):
    """Input, packed 3x3 weights and the prologue operands: G6D_PRO_CORR scales per position [H * W, cin] and shifts
    per channel, G6D_PRO_AFFINE(_RELU) per (group of group_rows images, channel)."""
    gen = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(B, H, W, cs or cin, generator=gen).cuda()
    w = torch.randn(cout, cin, 3, 3, generator=gen) * (2 / (9 * cin)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(cout, generator=gen).cuda(), pad=1)
    if pro == ops.PRO_CORR:
        ps, pb = torch.rand(H * W, cin, generator=gen) * 1.5 + 0.25, torch.randn(cin, generator=gen)
    else:
        groups = (B + group_rows - 1) // group_rows
        ps, pb = torch.rand(groups, cin, generator=gen) + 0.5, torch.randn(groups, cin, generator=gen) * 0.5
    return x, pc, ps.cuda(), pb.cuda()


def both(ops, x, pc, pro, ps, pb, group_rows, in_coff=0, stats_rows=None):
    """(prenormalised split input, producer warps) results of the same convolution."""
    kw = dict(prologue=pro, pro_scale=ps, pro_shift=pb, group_rows=group_rows, in_coff=in_coff, stats_rows=stats_rows)
    a = ops.conv(x, pc, prenorm=True, **kw)
    b = ops.conv(x, pc, **kw)
    torch.cuda.synchronize()
    return a, b


def check_plans(ops, x, pc, pro, group_rows, in_coff=0):
    from gen6d_b200 import _lib
    pre = plan(x, pc, pro, group_rows, _lib.TC_PRENORM, in_coff)
    gather = plan(x, pc, pro, group_rows, 0, in_coff)
    assert pre[0] == 0 and pre[3] == 1                     # persistent kernel, A by TMA im2col
    assert gather[3] == 0 and pre[:3] == gather[:3]        # same kernel, BN and K splits either way
    return pre


PROS = ['PRO_CORR', 'PRO_AFFINE', 'PRO_AFFINE_RELU']


# The selector towers' 8x8 and 4x4 layers.  A 128-row tile holds 2 images of 8x8 or 8 of 4x4; with groups of 3 images
# the tiles cross group boundaries.  The moments are one group over all rows, as in the towers.
@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('B, H, cin, cout, split_k', [
    (20, 8, 512, 128, True),        # K = 4608: split-K and the reduce kernel (with the fused moments)
    (320, 8, 128, 128, False),      # a tower layer's shape, one K split: moments fused into the kernel's epilogue
    (40, 4, 256, 256, True),        # Cout 256: two N tiles
    (320, 4, 512, 256, True),       # level 2's first layer
])
def test_prenorm_bit_identical(ops, pro, B, H, cin, cout, split_k):
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, B, H, H, cin, cout, pro, 3, seed=B * H + cin + cout + pro)
    _, bn, splits, _ = check_plans(ops, x, pc, pro, 3)
    assert bn == 128 and (splits > 1) == split_k
    rows = B * H * H
    (ya, sa), (yb, sb) = both(ops, x, pc, pro, ps, pb, 3, stats_rows=rows)
    assert torch.equal(ya, yb)
    assert float(ya.abs().max()) > 0
    # fp64 atomics from many CTAs over equal outputs: equal up to the order of the additions (a partial sum that
    # cancels to ~1e-7 of the total loses its last bits in a different place)
    np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('B, residue', [(63, 1), (64, 64), (65, 127)])
def test_prenorm_last_tile_residues(ops, pro, B, residue):
    """7 x 9 planes: M = 63 B leaves 1, 64 or 127 rows in the last tile; groups of 2 images."""
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, B, 7, 9, 64, 64, pro, 2, seed=B + 100 * pro)
    assert (B * 7 * 9) % 128 == residue
    assert check_plans(ops, x, pc, pro, 2)[1] == 64
    a, b = both(ops, x, pc, pro, ps, pb, 2)
    assert torch.equal(a, b)


@pytest.mark.parametrize('pro', PROS)
def test_prenorm_channel_slice(ops, pro):
    """Input channels [128, 256) of a 384-wide row: the prologue operands index the slice's channels."""
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, 12, 8, 8, 128, 128, pro, 5, seed=31 + pro, cs=384)
    check_plans(ops, x, pc, pro, 5, in_coff=128)
    a, b = both(ops, x, pc, pro, ps, pb, 5, in_coff=128)
    assert torch.equal(a, b)
