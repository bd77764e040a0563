"""G6D_TC_FOLD_SPLITS on the GPU: a folded layer (one CTA sums a tile's K splits in the output, in the split-K reduce's
order) must give the flag-less output bit for bit, and its fused moments up to the order of their fp64 additions.
Covered: 2, 3, 4 and 8 splits; the default K order and the A-reuse kernel's (reuse_im2col), 2-D and a 32^3 volume
(rank-5 im2col); BN 64 and 128; bias + ReLU or neither; with and without moments; M % 128 of 1, 64 and 127; an output
channel slice of an odd-strided buffer; the detector's correlation at 480 and 960 columns (one and two objects)."""
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


def plan(x, pc, flags, out_cstride):
    from gen6d_b200 import _lib
    if x.dim() == 4:
        (B, H, W, cs), D = x.shape, 1
    else:
        B, D, H, W, cs = x.shape
    (kd, kh, kw), (pd, ph, pw) = pc.k, pc.pad
    d = _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=0, Cout=pc.cout, kd=kd, kh=kh, kw=kw,
                      stride=1, pd=pd, ph=ph, pw=pw, Do=D + 2 * pd - kd + 1, Ho=H + 2 * ph - kh + 1, Wo=W + 2 * pw - kw + 1,
                      out_cstride=out_cstride, out_coff=0, prologue=0, group_rows=1, act=0, max_chain_k=pc.max_chain_k)
    out = (ctypes.c_int * 5)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_v2(ctypes.byref(d), pc.kind, flags, out, 5), 'g6d_conv_tc_plan_v2')
    return list(out)


def fold_vs_split(ops, x, pc, splits, ro, stats_rows=None, out_coff=None, **kw):
    """Runs the layer with and without fold_splits (same other flags), checks the plans, compares."""
    from gen6d_b200 import _lib
    flags = _lib.TC_REUSE_IM2COL if ro else 0
    ocs = pc.cout if out_coff is None else out_coff + pc.cout + 2
    p_fold, p_split = plan(x, pc, flags | _lib.TC_FOLD_SPLITS, ocs), plan(x, pc, flags, ocs)
    assert p_fold == p_split[:4] + [1] and p_split[4] == 0
    assert p_split[0] == 0 and p_split[2] == splits and p_split[3] == 1
    if ro:      # in the A-reuse kernel's K order: without reuse_im2col the A-reuse kernel would run
        assert plan(x, pc, 0, ocs)[0] == 1
    else:
        assert plan(x, pc, 0, ocs)[:4] == p_split[:4]
    res = []
    for fold in (True, False):
        if out_coff is None:
            r = ops.conv(x, pc, reuse_im2col=ro, fold_splits=fold, stats_rows=stats_rows, **kw)
        else:
            out = torch.full((*x.shape[:-1], ocs), float('nan'), device='cuda')
            r = ops.conv(x, pc, reuse_im2col=ro, fold_splits=fold, out=out, out_coff=out_coff, **kw)
            r = out
        res.append(r)
    torch.cuda.synchronize()
    (a, b) = res
    if stats_rows is not None:
        (a, sa), (b, sb) = a, b
        np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)
    if out_coff is not None:
        assert torch.isnan(a[..., :out_coff]).all() and torch.isnan(a[..., out_coff + pc.cout:]).all()
        a, b = a[..., out_coff:out_coff + pc.cout], b[..., out_coff:out_coff + pc.cout]
    assert torch.equal(a, b)
    assert float(a.abs().max()) > 0
    return a


def layer(ops, shape, cin, cout, k, seed, bias=True, max_chain_k=0):
    gen = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(*shape, cin, generator=gen).clamp_min(0).cuda()
    taps = k[0] * k[1] * k[2]
    w = torch.randn(cout, cin, *k, generator=gen) * (2 / (taps * cin)) ** .5
    b = torch.randn(cout, generator=gen).cuda() if bias else None
    pc = ops.pack_conv(w.cuda(), b, pad=1)
    pc.max_chain_k = max_chain_k
    return x, pc


# (B, H, W, Cin, Cout, max_chain_k, splits, A-reuse K order, bias + ReLU, moments): M = B H W with M % 128 of 1, 64, 127
CASES = [
    pytest.param(5, 129, 77, 256, 128, 0, 2, False, True, False, id='default-s2-bn128-m1'),
    pytest.param(5, 127, 77, 512, 128, 0, 3, False, True, False, id='default-s3-bn128-m127'),
    pytest.param(2, 124, 120, 512, 128, 0, 3, False, True, True, id='default-s3-bn128-m64-stats'),
    pytest.param(2, 124, 120, 512, 128, 640, 8, False, False, False, id='default-s8-bn128-m64-plain'),
    pytest.param(2, 124, 120, 256, 64, 192, 4, False, True, True, id='default-s4-bn64-m64-stats'),
    pytest.param(5, 127, 77, 256, 64, 256, 2, True, True, False, id='ro-s2-bn64-m127'),
    pytest.param(5, 129, 77, 256, 64, 256, 2, True, False, False, id='ro-s2-bn64-m1-plain'),
    pytest.param(3, 96, 90, 256, 64, 256, 2, True, True, True, id='ro-s2-bn64-m64-stats'),
]


@pytest.mark.parametrize('B, H, W, cin, cout, mck, splits, ro, relu, stats', CASES)
def test_fold_bit_identical(ops, B, H, W, cin, cout, mck, splits, ro, relu, stats):
    x, pc = layer(ops, (B, H, W), cin, cout, (1, 3, 3), seed=B * H * W + cin + cout + splits, bias=relu, max_chain_k=mck)
    fold_vs_split(ops, x, pc, splits, ro, stats_rows=H * W if stats else None, act=ops.ACT_RELU if relu else ops.ACT_NONE)


def test_fold_output_channel_slice(ops):
    """Columns [131, 259) of a 261-channel buffer: odd row stride, so every element is stored and re-read on its own."""
    x, pc = layer(ops, (2, 124, 120), 512, 128, (1, 3, 3), seed=11, max_chain_k=640)
    fold_vs_split(ops, x, pc, 8, False, out_coff=131, act=ops.ACT_RELU)


def test_fold_volume_32_256_64(ops):
    """A 32^3 volume, 256 -> 64 channels (BN 64): two splits on the rank-5 im2col map, with moments per volume."""
    x, pc = layer(ops, (1, 32, 32, 32), 256, 64, (3, 3, 3), seed=32)
    fold_vs_split(ops, x, pc, 2, True, stats_rows=32 ** 3)


def corr_kernels(ops, k, n_obj, gen, c=512, rfn=32):
    """Detector.pack_kernels' row-decomposed operand for n_obj objects' [rfn, k, k, c] post-ReLU reference maps."""
    feats = [torch.randn(rfn, k, k, c, generator=gen).clamp_min(0) for _ in range(n_obj)]
    flat = torch.cat([f.permute(1, 0, 2, 3).reshape(k * rfn, k * c) for f in feats], 0).contiguous().cuda()
    pc = ops.PackedConv(None, None, c, n_obj * k * rfn, (1, 1, k), 1, (0, k // 2, k // 2))
    pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, ops.tc_kind_for(c))
    pc.max_chain_k = 640
    return pc


# the 1 x 15 correlation at 1/8 of the 480 x 640 scale (8 splits; 480 and 960 columns) and the 1 x 7 one at 1/16 of the
# largest scale with two objects (4 splits)
@pytest.mark.parametrize('k, h, w, n_obj, splits', [(15, 60, 80, 1, 8), (15, 60, 80, 2, 8), (7, 44, 58, 2, 4)])
def test_fold_correlation(ops, k, h, w, n_obj, splits):
    gen = torch.Generator(device='cpu').manual_seed(10 * k + n_obj)
    x = torch.randn(10, h, w, 512, generator=gen).clamp_min(0).cuda()
    fold_vs_split(ops, x, corr_kernels(ops, k, n_obj, gen), splits, True)
