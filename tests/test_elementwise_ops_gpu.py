"""The shared layout, resize, pooling and normalisation kernels (csrc/elementwise.cu) on the GPU against float64
or exact float32 CPU restatements of the same operations, at the shapes where indexing goes wrong: groups split
over several blocks, groups of fewer than 32 rows, channel offsets inside a wider row, odd image sizes, channel
counts that are not a multiple of 32 or 128, padding channels, N > 1.

Tolerances are |got - want| <= atol + rtol*|want|, each derived in a comment; every check prints its worst error.
Where a kernel's fp32 arithmetic is fixed (one fma, one IEEE division), the restatement does the same operations
with the same roundings and the check is bit for bit."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from test_tail_ops_gpu import U, check, gen, ulp_gap

pytestmark = pytest.mark.gpu

SENTINEL = -7777.0
U64 = 2.0 ** -53


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


def fma32(a, b, c):
    """fmaf(a, b, c) for float32 tensors: a*b + c rounded once to float32 (round to nearest even).  The product is
    exact in float64 and TwoSum gives the exact error of the float64 sum, so the float64 result t is off only when
    it lands exactly halfway between two floats while the exact sum does not: the error's sign then picks the side."""
    a, b, c = a.double(), b.double(), c.double()
    p = a * b
    t = p + c
    bp = t - p
    err = (p - (t - bp)) + (c - bp)
    r = t.float()
    up = torch.nextafter(r, torch.full_like(r, math.inf))
    dn = torch.nextafter(r, torch.full_like(r, -math.inf))
    r = torch.where((t == (r.double() + up.double()) / 2) & (err > 0), up, r)
    r = torch.where((t == (r.double() + dn.double()) / 2) & (err < 0), dn, r)
    return r


def mul32(a, b):
    return (a.double() * b.double()).float()      # exact product, one rounding


def test_fma32_emulation_on_ties():
    """The emulation itself, on sums built to sit on a float32 midpoint in float64 while the exact value does not."""
    f = lambda v: torch.tensor([v], dtype=torch.float32)
    a, b = f(1 + 2.0 ** -23), f(2.0 ** -24 - 2.0 ** -47)               # a*b = 2^-24 - 2^-70, exact in float64
    c = f(1 + 2.0 ** -23)
    # exact a*b + c = (1 + 3 * 2^-24) - 2^-70, just below the midpoint between 1 + 2^-23 and 1 + 2^-22: rounds down.
    # In float64 the sum is the midpoint itself, and round-to-even then goes up.
    assert float((a.double() * b.double() + c.double()).float()) == 1 + 2.0 ** -22
    assert float(fma32(a, b, c)) == 1 + 2.0 ** -23
    assert float(fma32(a, -b, -c)) == -(1 + 2.0 ** -23)
    # the same on the other side of the midpoint, and an exact tie, which stays round-to-even
    assert float(fma32(a, f(2.0 ** -24), c)) == 1 + 2.0 ** -22
    assert float(fma32(f(1.0), f(3 * 2.0 ** -24), f(1.0))) == 1 + 2.0 ** -22


# ----------------------------------------------------------------------------------------------------------------------
# g6d_instnorm_stats / g6d_instnorm_partial + g6d_instnorm_finalize
# ----------------------------------------------------------------------------------------------------------------------
def stats_bound(xg, eps, chunk=32):
    """float64 (mean, rstd) of each (group, channel) of xg [groups, rows, C] and forward error bounds of the kernels'
    statistics, which sum fp32 partials of at most `chunk` consecutive rows (x sequentially, x^2 by fmas) and add the
    partials in float64:
        |d sum x|   <= ((chunk - 1) u + n 2^-53) sum |x|      |d sum x^2| <= (chunk u + n 2^-53) sum x^2
    so with n rows, dm = |d sum x| / n and dE2 = |d sum x^2| / n, the variance E[x^2] - mean^2 is within
        dv = dE2 + (2 |mean| + dm) dm + 4 2^-53 (E[x^2] + mean^2).
    dv grows with mean^2 against a variance that does not: relative to the variance it is ~ 3 chunk u (mean/std)^2.
    rstd = 1/sqrt(var + eps) then lies between the values at max(var - dv, 0) and var + dv, and rounds once to fp32;
    shift = -mean rstd moves by |mean| d rstd + dm rstd_max and a rounding."""
    x = xg.double()
    n = x.shape[1]
    mean = x.mean(1)
    var = x.var(1, unbiased=False)
    e2 = (x * x).mean(1)
    dm = ((chunk - 1) * U + n * U64) * x.abs().mean(1)
    de2 = (chunk * U + n * U64) * e2
    dv = de2 + (2 * mean.abs() + dm) * dm + 4 * U64 * (e2 + mean * mean)
    rstd = 1 / torch.sqrt(var + eps)
    r_hi = 1 / torch.sqrt((var - dv).clamp_min(0) + eps)
    r_lo = 1 / torch.sqrt(var + dv + eps)
    a_rstd = torch.maximum(r_hi - rstd, rstd - r_lo) + U * r_hi
    a_shift = mean.abs() * a_rstd + dm * r_hi + U * mean.abs() * r_hi
    return mean, rstd, a_rstd, a_shift, dv / (var + eps)


IN_CASES = [   # rows_per_group, groups, C, cstride, coff
    (1, 700, 4, 8, 4), (5, 700, 64, 64, 0), (31, 3, 100, 104, 4), (32, 3, 512, 512, 0), (33, 1, 64, 128, 64),
    (320, 1, 100, 100, 0), (320, 3, 4, 12, 8), (64 * 5, 700, 4, 4, 0), (2000, 3, 512, 516, 4),
]


@pytest.mark.parametrize('ratio', [0.0, 10.0, 100.0])
@pytest.mark.parametrize('rpg,groups,Cc,cstride,coff', IN_CASES)
def test_instnorm_stats_matches_fp64(ops, rpg, groups, Cc, cstride, coff, ratio):
    """x = mean + N(0, 1) per channel with mean / std = ratio, in channels [coff, coff + C) of rows of cstride (the rest
    NaN: never read).  Small groups put many groups on grid.y, large ones split a group over several blocks."""
    eps = 1e-5
    g = gen(rpg * 7 + groups + Cc + int(ratio))
    x = torch.full((groups * rpg, cstride), math.nan)
    mu = ratio * (1 + 0.1 * torch.rand(groups, 1, Cc, generator=g))
    xs = (mu + torch.randn(groups, rpg, Cc, generator=g)).reshape(-1, Cc)
    x[:, coff:coff + Cc] = xs
    xd = x.cuda()
    mean, rstd, a_rstd, a_shift, _ = stats_bound(xs.reshape(groups, rpg, Cc), eps)
    scale, shift = ops.instnorm_stats(xd, rpg, channels=Cc, coff=coff, eps=eps)
    name = f'instnorm rpg={rpg} groups={groups} C={Cc} coff={coff} mean/std={ratio:g}'
    check(name + ' rstd', scale.cpu(), rstd, a_rstd, 0.0)
    check(name + ' shift', shift.cpu(), -mean * rstd, a_shift, 0.0)
    ws = ops.instnorm_partial(xd, rpg, channels=Cc, coff=coff)
    s, sf = ops.instnorm_finalize(ws, rpg, eps)
    check(name + ' partial+finalize rstd', s.cpu(), rstd, a_rstd, 0.0)
    check(name + ' partial+finalize shift', sf.cpu(), -mean * rstd, a_shift, 0.0)


def _rel_rstd(got, rstd):
    return float(((got.cpu().double() - rstd).abs() / rstd).max())


def test_instnorm_conditioning_at_large_mean(ops):
    """The selector's first tower InstanceNorm3d runs over S*h*w = 320*16*16 = 81920 rows per channel.  At mean / std
    = 0, 10, 100 this prints the measured relative rstd error of instnorm_stats and its bound (the bound is asserted
    through the checks).  The bound's relative variance error is ~ 3 * 32 u (mean/std)^2: 6e-4 at 10, 6e-2 at 100."""
    eps, rpg, Cc = 1e-5, 81920, 64
    g = gen(81920)
    z = torch.randn(rpg, Cc, generator=g)
    for ratio in (0.0, 10.0, 100.0):
        xs = ratio + z
        mean, rstd, a_rstd, a_shift, rel_v = stats_bound(xs[None], eps)
        scale, shift = ops.instnorm_stats(xs.cuda(), rpg, eps=eps)
        check(f'instnorm 81920 rows mean/std={ratio:g} rstd', scale.cpu(), rstd, a_rstd, 0.0)
        check(f'instnorm 81920 rows mean/std={ratio:g} shift', shift.cpu(), -mean * rstd, a_shift, 0.0)
        print(f'instnorm_stats mean/std={ratio:g}: measured relative rstd error {_rel_rstd(scale, rstd):.3e}, '
              f'bound {float((a_rstd / rstd).max()):.3e} (relative variance bound {float(rel_v.max()):.3e})')


def test_conv_fused_moments_conditioning(ops):
    """The convolution epilogue's fused output moments: fp32 partials over at most 32 rows of one group, added in
    float64 (the same structure as instnorm_stats, so the same bound).  A 1x1 layer 64 -> 64 with weights ~ 1/sqrt(64)
    (outputs of unit spread) and a bias of mean/std = 0, 10, 100; 2 images of 128 x 128, one group per image.  The
    reference statistics are float64 over the layer's own fp32 output, so only the moments are under test."""
    from gen6d_b200 import _lib
    eps, B, H, W, cin, cout = 1e-5, 2, 128, 128, 64, 64
    rows = H * W
    g = gen(4242)
    x = torch.randn(B, H, W, cin, generator=g).cuda()
    w = (torch.randn(cout, cin, 1, 1, generator=g) / 8).cuda()
    jitter = torch.rand(cout, generator=g)
    for ratio in (0.0, 10.0, 100.0):
        b = (ratio * (1 + 0.1 * jitter)).cuda()
        pc = ops.pack_conv(w, b, pad=0)
        d = _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=pc.cin, in_cstride=cin, in_coff=0, Cout=cout, kd=1, kh=1, kw=1, stride=1,
                          pd=0, ph=0, pw=0, Do=1, Ho=H, Wo=W, out_cstride=cout, out_coff=0, prologue=0, group_rows=1, act=0,
                          max_chain_k=0)
        assert pc.w_hi is not None and _lib.lib().g6d_conv_tc_stats_supported(C.byref(d), pc.kind, rows), \
            'the layer must take the fused-moments epilogue'
        y, ws = ops.conv(x, pc, stats_rows=rows)
        scale, shift = ops.instnorm_finalize(ws, rows, eps)
        yg = y.cpu().reshape(B, rows, cout)
        mean, rstd, a_rstd, a_shift, _ = stats_bound(yg, eps)
        check(f'conv fused moments mean/std={ratio:g} rstd', scale.cpu(), rstd, a_rstd, 0.0)
        check(f'conv fused moments mean/std={ratio:g} shift', shift.cpu(), -mean * rstd, a_shift, 0.0)
        print(f'conv fused moments mean/std={ratio:g}: measured relative rstd error {_rel_rstd(scale, rstd):.3e}, '
              f'bound {float((a_rstd / rstd).max()):.3e}')


# ----------------------------------------------------------------------------------------------------------------------
# g6d_affine_act
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('act', [0, 1])
@pytest.mark.parametrize('rows,rpg,Cc,ics,ico,ocs,oco', [(35, 5, 4, 4, 0, 4, 0), (60, 20, 64, 72, 8, 128, 64),
                                                        (21, 7, 100, 104, 4, 100, 0), (8, 1, 512, 516, 4, 520, 8)])
def test_affine_act_bit_exact(ops, rows, rpg, Cc, ics, ico, ocs, oco, act):
    """out[r, oco + c] = act(fmaf(x[r, ico + c], scale[g, c], shift[g, c])), g = r // rpg, bit for bit against the
    emulated fmaf.  Also reported: how many elements the double-rounded float64 restatement (x*s exact, + b rounded
    to float64, then to float32) gets wrong, which the emulation's midpoint fix-up corrects."""
    g = gen(rows + Cc + ics + act)
    groups = rows // rpg
    x = torch.full((rows, ics), math.nan)
    x[:, ico:ico + Cc] = torch.randn(rows, Cc, generator=g)
    scale = 1 + torch.randn(groups, Cc, generator=g)
    shift = torch.randn(groups, Cc, generator=g)
    out = torch.full((rows, ocs), SENTINEL).cuda()
    ops.affine_act(x.cuda(), scale.cuda(), shift.cuda(), rpg, act=act, channels=Cc, in_coff=ico, out=out, out_coff=oco)
    got = out.cpu()
    gi = torch.arange(rows) // rpg
    xs = x[:, ico:ico + Cc]
    want = fma32(xs, scale[gi], shift[gi])
    naive = (xs.double() * scale[gi].double() + shift[gi].double()).float()
    if act == 1:
        want, naive = want.clamp_min(0), naive.clamp_min(0)
    n_naive = int((naive != want).sum())
    print(f'affine_act rows={rows} C={Cc} act={act}: max gap {ulp_gap(got[:, oco:oco + Cc], want)} ulp; double-rounded '
          f'float64 differs in {n_naive} of {want.numel()} elements')
    assert torch.equal(got[:, oco:oco + Cc], want)
    assert ulp_gap(naive, want) <= 1
    assert bool((got[:, :oco] == SENTINEL).all()) and bool((got[:, oco + Cc:] == SENTINEL).all())


# ----------------------------------------------------------------------------------------------------------------------
# g6d_resize_bilinear / g6d_resize_nearest
# ----------------------------------------------------------------------------------------------------------------------
def _src32(Ho, Hi):
    """bilinear_src in float32: scale = Hi/Ho (IEEE), s = fmaf(dst + 0.5, scale, -0.5) clamped at 0 (nvcc contracts
    scale*(dst+0.5) - 0.5 into one fma), i0 = trunc(s) <= Hi - 1, i1 = min(i0 + 1, Hi - 1), l = s - i0."""
    scale = torch.tensor([float(Hi)], dtype=torch.float32) / torch.tensor([float(Ho)], dtype=torch.float32)
    dst = torch.arange(Ho, dtype=torch.float32) + 0.5
    s = fma32(dst, scale.expand(Ho), torch.full((Ho,), -0.5)).clamp_min(0)
    i0 = s.long().clamp_max(Hi - 1)
    i1 = (i0 + 1).clamp_max(Hi - 1)
    l1 = s - i0.float()
    return i0, i1, l1, 1 - l1


def bilinear32(x, Ho, Wo):
    """The kernel's arithmetic on x [N, Hi, Wi, C] float32: ATen's association hy (hx v00 + lx v01) + ly (hx v10 +
    lx v11), contracted as fmaf(hy, fmaf(lx, v01, hx v00), ly fmaf(lx, v11, hx v10))."""
    N, Hi, Wi, Cc = x.shape
    y0, y1, ly, hy = _src32(Ho, Hi)
    x0, x1, lx, hx = _src32(Wo, Wi)
    v = lambda yi, xi: x[:, yi][:, :, xi]                                       # N, Ho, Wo, C
    e = lambda t, ax: t.reshape([-1 if i == ax else 1 for i in range(4)]).expand(N, Ho, Wo, Cc)
    LX, HX, LY, HY = e(lx, 2), e(hx, 2), e(ly, 1), e(hy, 1)
    top = fma32(LX, v(y0, x1), mul32(HX, v(y0, x0)))
    bot = fma32(LX, v(y1, x1), mul32(HX, v(y1, x0)))
    return fma32(HY, top, mul32(LY, bot))


BILINEAR_CASES = [(2, 30, 40, 15, 20, 8), (1, 30, 40, 44, 61, 4), (3, 16, 16, 64, 64, 12), (2, 32, 24, 128, 96, 4),
                  (1, 128, 128, 120, 120, 3), (2, 1, 1, 7, 5, 8), (1, 37, 53, 16, 16, 64)]


@pytest.mark.parametrize('N,Hi,Wi,Ho,Wo,Cc', BILINEAR_CASES)
def test_resize_bilinear_bit_exact(ops, N, Hi, Wi, Ho, Wo, Cc):
    """Down and up by non-integer ratios, x2 and x4, a 1-pixel input; bit for bit against the float32 restatement and
    within 1e-6 of torch's CPU F.interpolate (inputs in [0, 1)), then written into channels [coff, coff + C) of a
    wider row with the rest left as they were."""
    x = torch.rand(N, Hi, Wi, Cc, generator=gen(Hi * Wi + Ho + Cc))
    got = ops.resize_bilinear(x.cuda(), Ho, Wo).cpu()
    want = bilinear32(x, Ho, Wo)
    print(f'resize_bilinear {Hi}x{Wi} -> {Ho}x{Wo} C={Cc}: max gap {ulp_gap(got, want)} ulp')
    assert torch.equal(got, want)
    ref = F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
    check(f'resize_bilinear {Hi}x{Wi} -> {Ho}x{Wo} vs torch', got, ref, 1e-6, 0.0)
    coff, ocs = 4, Cc + 12
    out = torch.full((N, Ho, Wo, ocs), SENTINEL).cuda()
    ops.resize_bilinear(x.cuda(), Ho, Wo, out=out, out_coff=coff)
    out = out.cpu()
    assert torch.equal(out[..., coff:coff + Cc], want)
    assert bool((out[..., :coff] == SENTINEL).all()) and bool((out[..., coff + Cc:] == SENTINEL).all())


@pytest.mark.parametrize('N,Hi,Wi,Ho,Wo,Cc', [(2, 128, 128, 120, 120, 3), (1, 480, 640, 120, 120, 4),
                                              (2, 100, 100, 120, 120, 5), (1, 60, 80, 120, 160, 8)])
def test_resize_nearest_bit_exact(ops, N, Hi, Wi, Ho, Wo, Cc):
    """The detector's 120 x 120 reference resize from 128 and from a 480 x 640 frame, an upscale, and x2."""
    x = torch.randn(N, Hi, Wi, Cc, generator=gen(Hi + Wi + Cc))
    got = ops.resize_nearest(x.cuda(), Ho, Wo).cpu()
    want = F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode='nearest').permute(0, 2, 3, 1)
    assert torch.equal(got, want)


# ----------------------------------------------------------------------------------------------------------------------
# g6d_maxpool2x2, g6d_l2norm_channels
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,H,W', [(2, 7, 9), (1, 2, 3), (3, 15, 4)])
@pytest.mark.parametrize('Cc', [4, 64, 516])
def test_maxpool2x2_odd_sizes(ops, N, H, W, Cc):
    """Odd H and W: the last row / column is dropped (floor), as in F.max_pool2d."""
    x = torch.randn(N, H, W, Cc, generator=gen(H * W + Cc))
    got = ops.maxpool2x2(x.cuda()).cpu()
    want = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(got, want)


@pytest.mark.parametrize('Cc', [4, 36, 512])
def test_l2norm_channels_matches_fp64(ops, Cc):
    """y = x / max(|x|, eps), eps = 1e-12, per row.  Rows: random, all zero (must give zeros, not NaN), a norm of
    ~1e-7 (just above eps: sqrt(ss + eps) would be ~5x off) and a norm of ~1e-14 (below eps: the clamp).  The sum of
    squares is C/32 + 5 roundings deep per lane and shuffle tree, the square root and the division add one each:
    rtol = ((C/32 + 5) / 2 + 3) u."""
    eps = 1e-12
    g = gen(Cc)
    x = torch.randn(40, Cc, generator=g)
    x[3] = 0
    x[7] *= 1e-7 / math.sqrt(Cc)
    x[11] *= 1e-14 / math.sqrt(Cc)
    got = ops.l2norm_channels(x.cuda(), eps).cpu()
    xd = x.double()
    want = xd / xd.norm(dim=1, keepdim=True).clamp_min(eps)
    rows = torch.arange(40) != 3                      # the zero row is checked for exact zeros below
    check(f'l2norm C={Cc}', got[rows], want[rows], 0.0, ((Cc / 32 + 5) / 2 + 3) * U)
    assert bool((got[3] == 0).all())
    assert float(want[11].abs().max()) < 0.5, 'the tiny row is clamped by eps'


# ----------------------------------------------------------------------------------------------------------------------
# g6d_nchw_to_nhwc / g6d_nhwc_to_nchw
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,Cc,H,W,pad', [(2, 3, 7, 9, 1), (1, 33, 5, 13, 3), (3, 64, 6, 6, 0), (1, 100, 9, 5, 28)])
def test_layout_round_trip_and_padding(ops, N, Cc, H, W, pad):
    """H*W and C not multiples of the 32 x 32 tile.  nchw_to_nhwc with out_c = C + pad writes the padding channels as
    zeros (the buffer is NaN before); nhwc_to_nchw reads only the first C of in_c channels (the rest NaN)."""
    x = torch.randn(N, Cc, H, W, generator=gen(Cc * H + W))
    out = torch.full((N, H, W, Cc + pad), math.nan).cuda()
    xd = x.cuda()
    ops._call('g6d_nchw_to_nhwc', ops._p(xd), ops._p(out), N, Cc, H, W, Cc + pad, ops._stream())
    got = out.cpu()
    assert torch.equal(got[..., :Cc], x.permute(0, 2, 3, 1))
    assert bool((got[..., Cc:] == 0).all()), 'padding channels must be written as zeros'
    wide = torch.full((N, H, W, Cc + pad), math.nan)
    wide[..., :Cc] = x.permute(0, 2, 3, 1)
    back = ops.nhwc_to_nchw(wide.cuda(), channels=Cc).cpu()
    assert torch.equal(back, x)
    assert torch.equal(ops.nhwc_to_nchw(ops.nchw_to_nhwc(x.cuda())).cpu(), x)


# ----------------------------------------------------------------------------------------------------------------------
# g6d_preprocess_u8 / g6d_imagenet_norm
# ----------------------------------------------------------------------------------------------------------------------
MEAN = torch.tensor([0.485, 0.456, 0.406], dtype=torch.float32)
STD = torch.tensor([0.229, 0.224, 0.225], dtype=torch.float32)


@pytest.mark.parametrize('norm', [False, True])
@pytest.mark.parametrize('out_c', [3, 4])
def test_preprocess_u8_every_byte_bit_exact(ops, out_c, norm):
    """All 256 byte values in each channel (the three channels cycle through them with different phases): x / 255,
    then (x - mean) / std, every operation an IEEE float32 one (no fast math), so torch's float32 gives the same bits."""
    v = torch.arange(256, dtype=torch.uint8)
    img = torch.stack([v, v.roll(85), v.flip(0)], 1).reshape(16, 16, 3)
    got = ops.preprocess_u8(img.cuda(), out_c=out_c, imagenet_norm=norm).cpu()
    want = img.float() / 255
    if norm:
        want = (want - MEAN) / STD
    assert torch.equal(got[..., :3], want)
    if out_c == 4:
        assert bool((got[..., 3] == 0).all())


@pytest.mark.parametrize('in_c', [3, 4])
@pytest.mark.parametrize('out_c', [3, 4])
def test_imagenet_norm_bit_exact(ops, in_c, out_c):
    x = torch.rand(5, 7, 11, in_c, generator=gen(in_c * 4 + out_c))
    if in_c == 4:
        x[..., 3] = math.nan                                   # not read
    got = ops.imagenet_norm(x.cuda(), out_c=out_c).cpu()
    assert torch.equal(got[..., :3], (x[..., :3] - MEAN) / STD)
    if out_c == 4:
        assert bool((got[..., 3] == 0).all())
