"""G6D_TC_REUSE_IM2COL on the layers besides the refiner's that the A-reuse kernel takes without it, at bench.py's
shapes: the detector's row-decomposed correlation (1 and 2 objects), the selector's 16x16 level-0 tower (q(.)ref
prologue with a per-position scale, then InstanceNorm+ReLU, both with fused moments), the crops' VGG at 32^2 and 16^2,
the detector's 1/16 maps and its heads.  With the flag they run on the persistent kernel with TMA im2col A in the A-reuse
kernel's K order and K splits, so outputs must equal the flag-less ones bit for bit, and the moments up to the order
of their fp64 additions.  One recorded predict_batch (bench.py's batch of 10, 3 refinements) checks that no
tensor-core convolution of the step plans the A-reuse kernel any more."""
import ctypes
import os
import sys

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


def plan(x, pc, prologue, flags):
    from gen6d_b200 import _lib
    B, H, W, cs = x.shape
    kd, kh, kw = pc.k
    pd, ph, pw = pc.pad
    d = _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=0, Cout=pc.cout, kd=kd, kh=kh, kw=kw,
                      stride=1, pd=pd, ph=ph, pw=pw, Do=1, Ho=H + 2 * ph - kh + 1, Wo=W + 2 * pw - kw + 1,
                      out_cstride=pc.cout, out_coff=0, prologue=prologue, group_rows=B, act=0,
                      max_chain_k=pc.max_chain_k)
    out = (ctypes.c_int * 4)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_ex(ctypes.byref(d), pc.kind, flags, out), 'g6d_conv_tc_plan_ex')
    return list(out)


def both(ops, x, pc, **kw):
    """(reuse_im2col, without it) results of one convolution; checks the plans first."""
    from gen6d_b200 import _lib
    pro = kw.get('prologue', ops.PRO_NONE)
    flags = _lib.TC_PRENORM if pro else 0
    ro, ref = plan(x, pc, pro, flags | _lib.TC_REUSE_IM2COL), plan(x, pc, pro, flags)
    assert ref[0] == 1 and ref[3] == 0                    # without the flag: the A-reuse kernel
    assert ro[0] == 0 and ro[3] == 1                      # with it: persistent kernel, A by TMA im2col
    assert ro[1:3] == ref[1:3]
    a = ops.conv(x, pc, reuse_im2col=True, prenorm=bool(pro), **kw)
    b = ops.conv(x, pc, prenorm=bool(pro), **kw)
    torch.cuda.synchronize()
    return a, b, ro


def check(a, b, stats=False):
    if stats:
        (a, sa), (b, sb) = a, b
        np.testing.assert_allclose(sa.cpu().numpy(), sb.cpu().numpy(), rtol=1e-12, atol=1e-9)
    assert torch.equal(a, b)
    assert float(a.abs().max()) > 0


def corr_kernels(ops, k, n_obj, gen, c=512, rfn=32):
    """Detector.pack_kernels' row-decomposed operand for n_obj objects' [rfn, k, k, c] post-ReLU reference maps."""
    feats = [torch.randn(rfn, k, k, c, generator=gen).clamp_min(0) for _ in range(n_obj)]
    flat = torch.cat([f.permute(1, 0, 2, 3).reshape(k * rfn, k * c) for f in feats], 0).contiguous().cuda()
    pc = ops.PackedConv(None, None, c, n_obj * k * rfn, (1, 1, k), 1, (0, k // 2, k // 2))
    pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, ops.tc_kind_for(c))
    pc.max_chain_k = 640
    return pc


# each correlation level at the largest (704 x 928) and the smallest (256 x 320) query scale of the step: the 1/8, 1/16
# and 1/32 maps against 15, 7 and 3-row kernels
@pytest.mark.parametrize('n_obj', [1, 2])
@pytest.mark.parametrize('k, h, w', [(15, 88, 116), (15, 32, 40), (7, 44, 58), (7, 16, 20), (3, 22, 29), (3, 8, 10)])
def test_correlation_bit_identical(ops, n_obj, k, h, w):
    gen = torch.Generator(device='cpu').manual_seed(100 * k + h + n_obj)
    x = torch.randn(10, h, w, 512, generator=gen).clamp_min(0).cuda()
    pc = corr_kernels(ops, k, n_obj, gen)
    a, b, ro = both(ops, x, pc)
    if k == 15:
        assert ro[2] == 8                                 # K = 7680 in chains of 640: eight splits over channel blocks
    check(a, b)


def test_split_k_reduce_four_columns_bit_identical(ops):
    """The split-K reduce takes four columns per thread when Cout % 4 == 0.  The correlation's 480 columns (8 splits)
    must equal the first 480 of the same correlation with two more kernels (Cout 482: one column per thread), whose
    columns are computed by the same tiles; and an output slice at channel offset 2 (no 16-byte row alignment, stored
    column by column) must equal both."""
    gen = torch.Generator(device='cpu').manual_seed(5)
    x = torch.randn(10, 32, 40, 512, generator=gen).clamp_min(0).cuda()
    pc = corr_kernels(ops, 15, 1, gen)
    extra = torch.randn(2, 15 * 512, generator=gen).clamp_min(0).cuda()
    wide = ops.PackedConv(None, None, 512, 482, pc.k, 1, pc.pad, max_chain_k=640, kind=pc.kind)
    hi, lo, _ = ops.split_operand(extra, pc.kind)
    wide.w_hi, wide.w_lo = torch.cat([pc.w_hi, hi], 0), torch.cat([pc.w_lo, lo], 0)
    assert plan(x, pc, 0, 0)[2] == plan(x, wide, 0, 0)[2] == 8
    a = ops.conv(x, pc, reuse_im2col=True)
    b = ops.conv(x, wide, reuse_im2col=True)
    out = torch.zeros(*a.shape[:3], 484, device='cuda')
    ops.conv(x, pc, out=out, out_coff=2, reuse_im2col=True)
    torch.cuda.synchronize()
    assert torch.equal(a, b[..., :480])
    assert torch.equal(a, out[..., 2:482])
    assert float(a.abs().max()) > 0


def test_selector_level0_tower_bit_identical(ops):
    """512->64 with the q(.)ref prologue (per-position scale [16*16, 512], per-channel shift), moments over the whole
    tensor; then 64->64 with InstanceNorm+ReLU (group_rows = S), moments again."""
    S = 320
    gen = torch.Generator(device='cpu').manual_seed(3)
    ref = torch.randn(S, 16, 16, 512, generator=gen).cuda()
    ps = (torch.rand(256, 512, generator=gen) + 0.5).cuda()
    pb = (torch.randn(512, generator=gen) * 0.1).cuda()
    w = torch.randn(64, 512, 3, 3, generator=gen) * (2 / (9 * 512)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(64, generator=gen).cuda(), pad=1)
    rows = S * 256
    a, b, ro = both(ops, ref, pc, prologue=ops.PRO_CORR, pro_scale=ps, pro_shift=pb, group_rows=S, stats_rows=rows)
    assert ro[2] == 1
    check(a, b, stats=True)
    y, st = b
    sc, sh = ops.instnorm_finalize(st, rows, 1e-5)
    w = torch.randn(64, 64, 3, 3, generator=gen) * (2 / (9 * 64)) ** .5
    pc = ops.pack_conv(w.cuda(), torch.randn(64, generator=gen).cuda(), pad=1)
    a, b, _ = both(ops, y, pc, prologue=ops.PRO_AFFINE_RELU, pro_scale=sc, pro_shift=sh, group_rows=S, stats_rows=rows)
    check(a, b, stats=True)


def vgg_layer(ops, B, h, w, cin, cout, seed):
    gen = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(B, h, w, cin, generator=gen).clamp_min(0).cuda()
    wt = torch.randn(cout, cin, 3, 3, generator=gen) * (2 / (9 * cin)) ** .5
    return x, ops.pack_conv(wt.cuda(), torch.randn(cout, generator=gen).cuda(), pad=1)


# the refiner crops' VGG at 1/4 and 1/8 of 128^2 (70 crops), the detector's 1/16 maps at scales -1, -0.5 and 0 of a
# 480 x 640 query (and 1/8 at -1) and the detector heads' first layer at 1/8
@pytest.mark.parametrize('B, h, w, cin, cout', [
    (70, 32, 32, 128, 256), (70, 32, 32, 256, 256), (70, 16, 16, 256, 512), (70, 16, 16, 512, 512),
    (10, 16, 20, 512, 512), (10, 22, 30, 512, 512), (10, 30, 40, 512, 512), (10, 32, 40, 256, 512),
    (10, 60, 80, 64, 64),
])
def test_vgg_and_head_layers_bit_identical(ops, B, h, w, cin, cout):
    x, pc = vgg_layer(ops, B, h, w, cin, cout, seed=h * w + cin + cout)
    a, b, _ = both(ops, x, pc, act=ops.ACT_RELU)
    check(a, b)


def test_predict_batch_plans_no_a_reuse_kernel(ops):
    """Every tensor-core convolution of one bench step (recorded and replayed eagerly, as tools/conv_breakdown.py
    does) plans the persistent kernel."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
    try:
        import conv_breakdown
    finally:
        sys.path.pop(0)
    _, rec = conv_breakdown.record_step(10, 3)
    prof = ops.enable_profiling()
    with torch.no_grad():
        for fn, inputs in rec:
            fn(*inputs)
    tags = [c[3] for c in ops.collect_profile(prof)['#calls']]
    assert len(tags) > 100
    reuse = sorted({t for t in tags if ' reuse ' in f' {t} '})
    assert not reuse, reuse
    assert sum(t.endswith('-ro') for t in tags) > 0
