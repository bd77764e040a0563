"""The persistent kernel's split input (A tiles by TMA im2col from an fp16 hi/lo copy of the input) against its
producer warps (gather, split, swizzle, st.shared): the tiles are the same bytes by construction, so outputs
and fused moments must be equal bit for bit.  The producer path is forced with an identity prologue
(x * 1 + 0 == x), which takes the same descriptor off the split input."""
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


def plan(ops, x, pc, prologue, in_coff=0):
    from gen6d_b200 import _lib
    B, H, W, cs = x.shape
    p = pc.pad[1]
    d = _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=in_coff, Cout=pc.cout, kd=1, kh=3, kw=3,
                      stride=1, pd=0, ph=p, pw=p, Do=1, Ho=H, Wo=W, out_cstride=pc.cout, out_coff=0, prologue=prologue,
                      group_rows=B, act=ops.ACT_RELU, max_chain_k=0)
    out = (ctypes.c_int * 4)()
    _lib.check(_lib.lib().g6d_conv_tc_plan(ctypes.byref(d), pc.kind, out), 'g6d_conv_tc_plan')
    return list(out)


def both(ops, x, pc, in_coff=0, stats_rows=None):
    """(split input, producer warps) results of the same convolution."""
    one = torch.ones(1, pc.cin, device='cuda')
    zero = torch.zeros(1, pc.cin, device='cuda')
    B = x.shape[0]
    a = ops.conv(x, pc, act=ops.ACT_RELU, in_coff=in_coff, stats_rows=stats_rows)
    b = ops.conv(x, pc, prologue=ops.PRO_AFFINE, pro_scale=one, pro_shift=zero, group_rows=B, act=ops.ACT_RELU,
                 in_coff=in_coff, stats_rows=stats_rows)
    torch.cuda.synchronize()
    return a, b


def shape_for(residue, W, B):
    """H such that M = B * H * W leaves `residue` rows in the last 128-row tile."""
    for H in range(2, 200):
        if (B * H * W) % 128 == residue:
            return H
    raise AssertionError((residue, W, B))


# W = 131 keeps the halo out of the A-reuse kernel's shared memory (BN 64 too), so these run on the persistent kernel
@pytest.mark.parametrize('residue', [1, 64, 65, 127])
@pytest.mark.parametrize('cin, cout', [(64, 128), (256, 128), (64, 64), (256, 64)])   # BN 128 / 64, K = 576 / 2304
def test_split_input_bit_identical(ops, residue, cin, cout):
    B, W = 3, 131
    H = shape_for(residue, W, B)
    gen = torch.Generator(device='cpu').manual_seed(residue * 1000 + cin + cout)
    x = torch.randn(B, H, W, cin, generator=gen).cuda()
    w = torch.randn(cout, cin, 3, 3, generator=gen) * (2 / (9 * cin)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(cout, generator=gen).cuda(), pad=1)
    kernel, bn, splits, split_in = plan(ops, x, pc, ops.PRO_NONE)
    assert (kernel, split_in) == (0, 1) and bn == (128 if cout > 64 else 64)
    assert plan(ops, x, pc, ops.PRO_AFFINE)[3] == 0
    if cin == 256 and cout == 128:
        assert splits > 1                                   # K = 2304 > 2048 at BN 128: split-K and the reduce kernel
    a, b = both(ops, x, pc)
    assert torch.equal(a, b)
    assert float(a.abs().max()) > 0


def test_split_input_channel_slice_and_batch(ops):
    """Input channels [64, 192) of a 256-wide row, B = 5 images of 11 x 83: tiles cross rows and images."""
    gen = torch.Generator(device='cpu').manual_seed(7)
    x = torch.randn(5, 11, 83, 256, generator=gen).cuda()
    w = torch.randn(128, 128, 3, 3, generator=gen) * (2 / (9 * 128)) ** .5
    pc = ops.pack_conv(w.cuda(), None, pad=1)
    assert plan(ops, x, pc, ops.PRO_NONE, in_coff=64)[3] == 1
    a, b = both(ops, x, pc, in_coff=64)
    assert torch.equal(a, b)


@pytest.mark.parametrize('cin', [64, 512])
def test_split_input_fused_moments(ops, cin):
    """Fused InstanceNorm moments (one group per image): outputs equal, moments equal up to atomic order."""
    B, H, W = 3, 6, 96                                      # H * W = 576 rows per group, a multiple of 32
    gen = torch.Generator(device='cpu').manual_seed(cin)
    x = torch.randn(B, H, W, cin, generator=gen).cuda()
    w = torch.randn(128, cin, 3, 3, generator=gen) * (2 / (9 * cin)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(128, generator=gen).cuda(), pad=1)
    assert plan(ops, x, pc, ops.PRO_NONE)[3] == 1
    (ya, sa), (yb, sb) = both(ops, x, pc, stats_rows=H * W)
    assert torch.equal(ya, yb)
    # fp64 atomics from many CTAs: equal up to the order of the additions
    np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)
