"""GPU parity of the individual C-ABI kernels against plain torch fp32 CPU references.
Tolerances are fp32 accumulation-order tolerances (stated per test)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def g(seed):
    gen = torch.Generator(device='cpu')
    gen.manual_seed(seed)
    return gen


def nhwc(x):   # NC(D)HW cpu -> channels-last cuda
    nd = x.dim()
    return x.permute(0, *range(2, nd), 1).contiguous().cuda()


def nchw(x):   # channels-last cuda -> NC(D)HW cpu
    nd = x.dim()
    return x.permute(0, nd - 1, *range(1, nd - 1)).contiguous().cpu()


def close(a, b, rtol=1e-4, atol=1e-4):
    np.testing.assert_allclose(a.detach().cpu().numpy(), b.detach().cpu().numpy(), rtol=rtol, atol=atol)


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


@pytest.mark.parametrize('B,H,W,cin,cout,act', [(2, 17, 23, 64, 64, 1), (1, 32, 40, 128, 256, 0), (3, 8, 8, 512, 32, 2),
                                                (1, 9, 7, 4, 64, 1), (2, 5, 5, 192, 2, 0), (1, 60, 80, 64, 1, 0)])
def test_conv2d_3x3(ops, B, H, W, cin, cout, act):
    x = torch.randn(B, cin, H, W, generator=g(1))
    w = torch.randn(cout, cin, 3, 3, generator=g(2)) * (2 / (9 * cin)) ** .5
    b = torch.randn(cout, generator=g(3))
    ref = F.conv2d(x, w, b, padding=1)
    ref = F.relu(ref) if act == 1 else (F.leaky_relu(ref, 0.1) if act == 2 else ref)
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    y = ops.conv(nhwc(x), pc, act=act)
    close(nchw(y), ref)


@pytest.mark.parametrize('stride', [1, 2])
def test_conv3d_3x3x3(ops, stride):
    x = torch.randn(2, 64, 8, 8, 8, generator=g(4))
    w = torch.randn(128, 64, 3, 3, 3, generator=g(5)) * (2 / (27 * 64)) ** .5
    b = torch.randn(128, generator=g(6))
    ref = F.conv3d(x, w, b, stride=stride, padding=1)
    y = ops.conv(nhwc(x), ops.pack_conv(w.cuda(), b.cuda(), stride=stride, pad=1))
    close(nchw(y), ref)


def test_conv_splitk_large_kernel(ops):
    """Detector-style correlation: 15x15x512 'kernels' over a small map -> split-K path."""
    q = torch.randn(1, 512, 12, 16, generator=g(7))
    r = torch.randn(5, 512, 15, 15, generator=g(8))
    ref = F.conv2d(q, r, padding=7)
    rk = r.permute(0, 2, 3, 1).contiguous().cuda()     # [rfn, k, k, c] channels-last features
    w = ops.transpose_to_packed(rk.reshape(5, -1))
    pc = ops.PackedConv(w, None, 512, 5, (1, 15, 15), 1, (0, 7, 7))
    y = ops.conv(nhwc(q), pc)
    close(nchw(y), ref, rtol=1e-4, atol=2e-2)


def test_conv_1x1_padded_cin_and_offsets(ops):
    x = torch.randn(40, 515, generator=g(9))
    w = torch.randn(512, 515, 1, generator=g(10)) * 0.05
    b = torch.randn(512, generator=g(11))
    ref = F.linear(x, w[:, :, 0], b)
    xin = torch.zeros(40, 516)
    xin[:, :515] = x
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=0, cin_pad=516)
    out = torch.zeros(40, 1, 1, 640, device='cuda')
    ops.conv(xin.cuda().reshape(40, 1, 1, 516), pc, out=out, out_coff=64)
    close(out.reshape(40, 640)[:, 64:576], ref)
    assert float(out.reshape(40, 640)[:, :64].abs().max()) == 0.0


@pytest.mark.parametrize('relu', [False, True])
def test_conv_affine_prologue_respects_zero_padding(ops, relu):
    """InstanceNorm(+ReLU) folded into the loader must equal norm -> pad -> conv."""
    x = torch.randn(3, 64, 10, 12, generator=g(12)) * 2 + 1
    w = torch.randn(32, 64, 3, 3, generator=g(13)) * 0.05
    xn = F.instance_norm(x)
    xn = F.relu(xn) if relu else xn
    ref = F.conv2d(xn, w, None, padding=1)
    xc = nhwc(x)
    ps, pb = ops.instnorm_stats(xc, rows_per_group=10 * 12)
    y = ops.conv(xc, ops.pack_conv(w.cuda(), None, pad=1), prologue=ops.PRO_AFFINE_RELU if relu else ops.PRO_AFFINE,
                 pro_scale=ps, pro_shift=pb, group_rows=1)
    close(nchw(y), ref, atol=2e-4)


def test_instnorm_stats_grouped(ops):
    x = torch.randn(6, 128, 7, 9, generator=g(14)) * 3 - 2     # selector style: one group over all 6 slices
    xr = x.permute(1, 0, 2, 3).reshape(1, 128, 6, 7, 9)
    ref = F.instance_norm(xr).reshape(128, 6, 7, 9).permute(1, 0, 2, 3)
    xc = nhwc(x)
    ps, pb = ops.instnorm_stats(xc, rows_per_group=6 * 7 * 9)
    y = ops.affine_act(xc, ps, pb, rows_per_group=6 * 7 * 9)
    close(nchw(y), ref, atol=1e-5)


def test_resize_pool_norm(ops):
    x = torch.rand(2, 8, 30, 40, generator=g(15))
    xc = nhwc(x)
    for size in ((15, 20), (44, 61), (60, 80), (30, 40)):
        close(nchw(ops.resize_bilinear(xc, *size)), F.interpolate(x, size=size, mode='bilinear'), atol=1e-6)
    close(nchw(ops.resize_nearest(xc, 28, 37)), F.interpolate(x, size=(28, 37)), atol=0)
    close(nchw(ops.maxpool2x2(xc)), F.max_pool2d(x, 2, 2), atol=0)
    close(nchw(ops.l2norm_channels(xc)), F.normalize(x, dim=1), atol=1e-7)
    img = (torch.rand(2, 16, 16, 3, generator=g(16)) * 255).to(torch.uint8)
    mean = torch.tensor([0.485, 0.456, 0.406]); std = torch.tensor([0.229, 0.224, 0.225])
    ref = (img.float() / 255 - mean) / std
    out = ops.preprocess_u8(img.cuda(), out_c=4, imagenet_norm=True)
    close(out[..., :3], ref, atol=1e-6)
    assert float(out[..., 3].abs().max()) == 0
    close(ops.nhwc_to_nchw(ops.nchw_to_nhwc(x.cuda())), x, atol=0)


def test_sel_corr_score_and_prologue(ops):
    S, P, Cc = 12, 64, 512
    ref = F.normalize(torch.rand(S, P, Cc, generator=g(17)), dim=2)
    q = F.normalize(torch.rand(P, Cc, generator=g(18)), dim=1)
    s = torch.einsum('pc,spc->sp', q, ref)
    want = torch.sum(s * (s / s.max(1, keepdim=True)[0]), 1)
    got = ops.sel_corr_score(ref.cuda(), q.cuda())
    close(got, want, rtol=1e-5, atol=1e-6)
    # closed-form first InstanceNorm3d of the correlation volume
    corr = (q[None] * ref).permute(2, 0, 1).reshape(1, Cc, S * P)      # [1, C, S*P]
    mean, var = corr.mean(2)[0], corr.var(2, unbiased=False)[0]
    s1, s2 = ops.sel_ref_sums(ref.cuda())
    scale, shift = ops.sel_corr_prologue(q.cuda(), s1, s2, S)
    rstd = 1 / torch.sqrt(var + 1e-5)
    close(shift, -mean * rstd, rtol=1e-4, atol=1e-5)
    close(scale, q * rstd[None], rtol=1e-4, atol=1e-6)


def test_sel_corr_score3_matches_per_level(ops):
    S = 10
    refs = [F.normalize(torch.rand(S, P, 512, generator=g(30 + i)), dim=2) for i, P in enumerate((256, 64, 16))]
    qs = [F.normalize(torch.rand(P, 512, generator=g(40 + i)), dim=1) for i, P in enumerate((256, 64, 16))]
    got = ops.sel_corr_score3([r.cuda() for r in refs], [q.cuda() for q in qs])        # dots + finish launches
    for l in range(3):
        s = torch.einsum('pc,spc->sp', qs[l], refs[l])
        want = torch.sum(s * (s / s.max(1, keepdim=True)[0]), 1)
        close(got[l], want, rtol=1e-5, atol=1e-6)
    # one launch: the CTA that completes a slice reduces it; the counters come back zero, call after call
    counters = torch.zeros(3 * S, dtype=torch.int32, device='cuda')
    for _ in range(3):
        fused = ops.sel_corr_score3([r.cuda() for r in refs], [q.cuda() for q in qs], counters=counters)
        assert torch.equal(fused, got)
        assert int(counters.abs().sum()) == 0


@pytest.mark.parametrize('S', [1, 7, 320])
def test_sel_corr_score3_fused_ragged_sizes(ops, S):
    """Odd slice counts / location counts that do not divide the per-CTA chunk."""
    Ps = (25, 9, 4)
    refs = [torch.rand(S, P, 512, generator=g(60 + i)).cuda() for i, P in enumerate(Ps)]
    qs = [torch.rand(P, 512, generator=g(70 + i)).cuda() for i, P in enumerate(Ps)]
    counters = torch.zeros(3 * S, dtype=torch.int32, device='cuda')
    a = ops.sel_corr_score3(refs, qs)
    b = ops.sel_corr_score3(refs, qs, counters=counters)
    assert torch.equal(a, b) and int(counters.abs().sum()) == 0


def test_attention_layernorm(ops):
    n, Cc, heads = 24, 512, 8
    q, k, v = [torch.randn(n, Cc, generator=g(19 + i)) for i in range(3)]
    r = lambda t: t.T.reshape(1, Cc // heads, heads, n)
    scores = torch.einsum('bdhn,bdhm->bhnm', r(q), r(k)) / (Cc // heads) ** .5
    want = torch.einsum('bhnm,bdhm->bdhn', torch.softmax(scores, -1), r(v)).reshape(Cc, n).T
    close(ops.attention(q.cuda(), k.cuda(), v.cuda(), heads), want, atol=1e-5)
    gam, bet = torch.rand(Cc, generator=g(23)), torch.rand(Cc, generator=g(24))
    close(ops.layernorm(q.cuda(), gam.cuda(), bet.cuda()), F.layer_norm(q, (Cc,), gam, bet), atol=1e-5)


@pytest.mark.parametrize('n', [5, 64, 100, 512])
def test_attention_head_major_tiled(ops, n):
    """The tiled kernel on head-major channels (c = head*64 + d) equals the reference-order kernel on the
    permuted tensors, and torch: attention.py:4-17 at n = 64 (one GPU) ... 512 (references over 8 GPUs)."""
    Cc, heads, D = 512, 8, 64
    q, k, v = [torch.randn(n, Cc, generator=g(80 + i)) for i in range(3)]
    r = lambda t: t.T.reshape(1, D, heads, n)
    scores = torch.einsum('bdhn,bdhm->bhnm', r(q), r(k)) / D ** .5
    want = torch.einsum('bhnm,bdhm->bdhn', torch.softmax(scores, -1), r(v)).reshape(Cc, n).T        # reference channel order
    hm = torch.arange(Cc)
    hm = (hm % D) * heads + hm // D                          # head-major position c' <- reference channel
    got = ops.attention(q[:, hm].contiguous().cuda(), k[:, hm].contiguous().cuda(), v[:, hm].contiguous().cuda(), heads, head_major=True)
    close(got, want[:, hm], atol=1e-5)
    close(got, ops.attention(q.cuda(), k.cuda(), v.cuda(), heads)[:, hm.cuda()], atol=1e-5)


_SMALLM_ACTS = {0: lambda y: y, 1: F.relu, 2: lambda y: F.leaky_relu(y, 0.1)}      # ACT_NONE, ACT_RELU, ACT_LEAKY01


def test_linear_smallm(ops):
    """linear_smallm against float64 at the refiner's regressor shapes: M in {1, 7, 8} poses (the kernel's limit is 8),
    K in {4, 512, 32768} (32768 is the flattened volume encoding), N in {1, 512}, every activation, plus the original
    M = 3, K = 4096, N = 64 leaky case.  Weights ~ 1/sqrt(K) keep the outputs O(1), where the fp32 dot of K terms is
    well inside the 1e-4 tolerance.  Every case runs; the failing ones are listed together."""
    cases = [(3, 4096, 64, ops.ACT_LEAKY01, 0.02)] + [(M, K, N, act, K ** -.5) for M in (1, 7, 8) for K in (4, 512, 32768)
                                                       for N in (1, 512) for act in (ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LEAKY01)]
    failed = []
    for M, K, N, act, wscale in cases:
        x = torch.randn(M, K, generator=g(25)); w = torch.randn(N, K, generator=g(26)) * wscale
        b = torch.randn(N, generator=g(27))
        want = _SMALLM_ACTS[act](F.linear(x.double(), w.double(), b.double()))
        got = ops.linear_smallm(x.cuda(), w.cuda(), b.cuda(), act=act)
        try:
            close(got, want)
        except AssertionError as e:
            failed.append(f'M={M} K={K} N={N} act={act}: {str(e).strip().splitlines()[-1]}')
    assert not failed, f'{len(failed)} of {len(cases)} cases out of tolerance:\n' + '\n'.join(failed)


@pytest.mark.parametrize('B,H,W', [(1, 64, 96), (3, 18, 22), (2, 128, 128)])
def test_vgg_first_block_fused_equals_conv_relu_pool(ops, B, H, W):
    """g6d_vgg_first_block (3x3 conv 4->64 + ReLU + 2x2 max-pool in one kernel) is bit-identical to the
    three separate kernels and matches torch."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 3, H, W, generator=g)
    w = torch.randn(64, 3, 3, 3, generator=g) * 0.2
    b = torch.randn(64, generator=g) * 0.1
    x4 = torch.zeros(B, H, W, 4)
    x4[..., :3] = x.permute(0, 2, 3, 1)
    x4 = x4.cuda()
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    fused = ops.vgg_first_block(x4, pc)
    sep = ops.maxpool2x2(ops.conv(x4, pc, act=ops.ACT_RELU))
    assert torch.equal(fused, sep)
    want = F.max_pool2d(F.relu(F.conv2d(x, w, b, padding=1)), 2).permute(0, 2, 3, 1)
    np.testing.assert_allclose(fused.cpu().numpy(), want.numpy(), atol=2e-5)
