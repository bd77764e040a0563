"""G6D_TC_REUSE_IM2COL against the kernels the same layers take without it.  Layers the A-reuse kernel would take run on
the persistent kernel with TMA im2col A, in the A-reuse kernel's K order and K splits; 3-D layers already on the
persistent kernel get the split input through the rank-5 map instead of the producer warps.  Every output element
sums the same products into the same accumulators in the same order, so outputs (and split-K partials, through the
reduce kernel) must be equal bit for bit, and the fused moments up to the order of their fp64 atomic additions."""
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


def plan(x, pc, prologue, flags, in_coff=0):
    from gen6d_b200 import _lib
    if x.dim() == 4:
        B, H, W, cs = x.shape
        D = 1
    else:
        B, D, H, W, cs = x.shape
    kd, kh, kw = pc.k
    pd, ph, pw = pc.pad
    d = _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=in_coff, Cout=pc.cout, kd=kd, kh=kh, kw=kw,
                      stride=1, pd=pd, ph=ph, pw=pw, Do=D, Ho=H, Wo=W, out_cstride=pc.cout, out_coff=0, prologue=prologue,
                      group_rows=1, act=0, max_chain_k=pc.max_chain_k)
    out = (ctypes.c_int * 4)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_ex(ctypes.byref(d), pc.kind, flags, out), 'g6d_conv_tc_plan_ex')
    return list(out)


def layer(ops, B, S, cin, cout, seed, D=None, cs=None):
    """Input [B, D, S, S, cs] (D = S; D = 1: a 2-D [B, S, S, cs] plane), packed 3^3 (3^2) weights and per-image
    InstanceNorm+ReLU operands."""
    gen = torch.Generator(device='cpu').manual_seed(seed)
    D = S if D is None else D
    shape = (B, S, S, cs or cin) if D == 1 else (B, D, S, S, cs or cin)
    k = (3, 3) if D == 1 else (3, 3, 3)
    x = torch.randn(*shape, generator=gen).cuda()
    w = torch.randn(cout, cin, *k, generator=gen) * (2 / (27 * cin)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(cout, generator=gen).cuda(), pad=1)
    ps, pb = torch.rand(B, cin, generator=gen) + 0.5, torch.randn(B, cin, generator=gen) * 0.5
    return x, pc, ps.cuda(), pb.cuda()


def both(ops, x, pc, pro, ps, pb, in_coff=0, stats_rows=None):
    """(REUSE_IM2COL, without it) results of the same convolution, prenorm on in both."""
    from gen6d_b200 import _lib
    flags = _lib.TC_PRENORM | _lib.TC_REUSE_IM2COL
    ro, ref = plan(x, pc, pro, flags, in_coff), plan(x, pc, pro, _lib.TC_PRENORM, in_coff)
    assert ro[0] == 0 and ro[3] == 1                      # persistent kernel, A by TMA im2col
    assert ro[1:3] == ref[1:3]                            # BN and K splits of the kernel it replaces
    kw = dict(prologue=pro, pro_scale=ps if pro else None, pro_shift=pb if pro else None, group_rows=1, in_coff=in_coff,
              stats_rows=stats_rows, prenorm=True)
    a = ops.conv(x, pc, reuse_im2col=True, **kw)
    b = ops.conv(x, pc, **kw)
    torch.cuda.synchronize()
    return (a, b), ro, ref


def check(a, b, stats=False):
    if stats:
        (a, sa), (b, sb) = a, b
        np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)
    assert torch.equal(a, b)
    assert float(a.abs().max()) > 0


PROS = ['PRO_NONE', 'PRO_AFFINE_RELU']


# The refiner's 3-D layers: the 32^3 embeds and trunk conv0 (A-reuse kernel; K = 6912 for Cin 256 splits over channel
# blocks and goes through the reduce kernel), trunk conv2 at 16^3 (A-reuse), conv4 at 8^3 and conv5.3 at 4^3
# (persistent; a tile spans two z-planes at 8^3 and two volumes at 4^3).
@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('B, S, cin, cout, kernel', [
    (2, 32, 256, 64, 1), (2, 32, 128, 64, 1), (2, 32, 64, 64, 1), (2, 16, 128, 128, 1),
    (3, 8, 256, 256, 0), (3, 4, 512, 512, 0),
])
def test_reuse_im2col_3d_bit_identical(ops, pro, B, S, cin, cout, kernel):
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, B, S, cin, cout, seed=S * cin + cout + pro)
    (a, b), ro, ref = both(ops, x, pc, pro, ps, pb, stats_rows=S ** 3)
    assert ref[0] == kernel
    if cin == 256 and S == 32:
        assert ro[2] > 1                                  # split-K partials through the reduce kernel
    check(a, b, stats=True)


# The feature branches over 70 crops: conv0 and conv_out at 32^2, conv1 at 16^2 (A-reuse kernel)
@pytest.mark.parametrize('pro', PROS)
@pytest.mark.parametrize('S, cin, cout', [(32, 256, 64), (32, 64, 64), (32, 192, 128), (32, 128, 128),
                                          (16, 512, 256), (16, 256, 64)])
def test_reuse_im2col_2d_branches_bit_identical(ops, pro, S, cin, cout):
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, 70, S, cin, cout, seed=S + cin + cout + pro, D=1)
    (a, b), ro, ref = both(ops, x, pc, pro, ps, pb, stats_rows=S * S)
    assert ref[0] == 1
    check(a, b, stats=True)


def test_reuse_im2col_max_chain_split(ops):
    """A shorter accumulate-chain bound: more splits over channel blocks, all through the reduce kernel."""
    x, pc, ps, pb = layer(ops, 1, 16, 512, 128, seed=7)
    pc.max_chain_k = 1024
    (a, b), ro, _ = both(ops, x, pc, ops.PRO_AFFINE_RELU, ps, pb)
    assert ro[2] >= 4
    check(a, b)


@pytest.mark.parametrize('pro', PROS)
def test_reuse_im2col_channel_slice(ops, pro):
    """Input channels [64, 192) of a 192-wide volume row (the trunk reading the embeds' concatenation)."""
    pro = getattr(ops, pro)
    x, pc, ps, pb = layer(ops, 2, 16, 128, 64, seed=11 + pro, cs=192)
    (a, b), _, _ = both(ops, x, pc, pro, ps, pb, in_coff=64)
    check(a, b)
