"""The networks' fused tail kernels (the volume fill, the detector's score fuse, the selector's vp_norm /
max-over-angles / parse, the pooled affine and the pose heads) on the GPU against float64 CPU
restatements of the same operations, at every instantiation and at the shapes where indexing goes wrong:
reference counts that are not the production 6, channel counts that are not a multiple of 128, grids
that are not a multiple of the 2x4x8 brick, non-square images, more than one 64-reference chunk.

A tolerance here is |got - want| <= atol + rtol*|want|, each stated with the fp32 operation count and
data magnitude it comes from; every check prints the worst error it saw.  Where two kernel paths do the
same fp32 arithmetic the check is bit for bit."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import gen6d_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


def gen(seed):
    return torch.Generator(device='cpu').manual_seed(seed)


def check(name, got, want, atol, rtol):
    """|got - want| <= atol + rtol*|want| elementwise (atol may be a tensor broadcast against want)."""
    got = got.detach().cpu().double()
    want = want.detach().cpu().double()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = (got - want).abs()
    lim = atol + rtol * want.abs()
    worst = float(err.max()) if err.numel() else 0.0
    frac = float((err / lim).max()) if err.numel() else 0.0
    print(f'{name}: worst |got - want| = {worst:.3e} ({frac:.3g} of the tolerance)')
    bad = ~(err <= lim)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f'{name}: {int(bad.sum())} of {err.numel()} elements out of tolerance; first at flat index {i}: '
                             f'got {got.flatten()[i].item()!r} want {want.flatten()[i].item()!r}; worst error {worst:.3e}')


def ulp_gap(a, b):
    """Largest distance in fp32 units in the last place between two float32 tensors of the same shape."""
    ia = a.detach().cpu().contiguous().view(torch.int32).long()
    ib = b.detach().cpu().contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7fffffff), ia)      # sign-magnitude -> a monotone integer line
    ib = torch.where(ib < 0, -(ib & 0x7fffffff), ib)
    return int((ia - ib).abs().max()) if ia.numel() else 0


# ----------------------------------------------------------------------------------------------------------------------
# g6d_ref_volume_fill
# ----------------------------------------------------------------------------------------------------------------------
SQUARE = (128, 128, 32, 32)      # img_h, img_w, fh, fw: the refiner's production sizes
WIDE = (96, 128, 24, 32)         # non-square image and feature map (a swapped h / w shows)
FOCAL = 100.0                    # the unit cube at depth ~3 spans the image and part of its border


def _rot(g):
    q = torch.randn(4, generator=g, dtype=torch.float64)
    w, x, y, z = (q / q.norm()).tolist()
    return torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                         [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                         [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)


def _pose(R, t):
    return torch.cat([R, torch.tensor(t, dtype=torch.float64)[:, None]], 1)


def volume_problem(Q, R, Cc, sn, size, seed):
    """Features N(0,1) and cameras for Q poses.  The poses differ per query; for query 0, reference view 0 has part of
    the cube behind its camera (the pz < 1e-4 clamp) and, with R >= 3, view R-1 looks at it from the side, so that some
    voxels project well off the feature map (the close_by guard).  Every view sees part of the cube off the image
    (zero padding and partial border taps).  Returned as the fp32 tensors the kernel takes."""
    img_h, img_w, fh, fw = size
    g = gen(seed)
    K = torch.tensor([[FOCAL, 0, img_w / 2], [0, FOCAL, img_h / 2], [0, 0, 1]], dtype=torch.float64)
    que_poses, ref_poses = [], []
    for q in range(Q):
        que_poses.append(_pose(_rot(g), [0.2 * float(torch.randn(1, generator=g)), 0.2 * float(torch.randn(1, generator=g)), 3.0]))
        refs = []
        for v in range(R):
            t = [0.3 * float(torch.randn(1, generator=g)), 0.3 * float(torch.randn(1, generator=g)),
                 3.0 + 0.3 * float(torch.randn(1, generator=g))]
            Rv = _rot(g)
            if q == 0 and v == 0:
                # camera 1 unit from the cube centre: z_c = Z + 1 < 0 for part of the cube.  x_c = X + 3 >= 1.27 there,
                # so px = f x_c + c_x z_c > 0 and the clamped voxels land ~1e6 pixels off the image, far from any tap
                Rv, t = torch.eye(3, dtype=torch.float64), [3.0, 0.0, 1.0]
            elif q == 0 and v == R - 1 and R >= 3:
                t = [2.5, 0.0, 3.0]
            refs.append(_pose(Rv, t))
        ref_poses.append(torch.stack(refs))
    f32 = lambda t: t.float().contiguous()
    return dict(ref_feats=torch.randn(Q, R, fh, fw, Cc, generator=g), que_feats=torch.randn(Q, fh, fw, Cc, generator=g),
                ref_Ks=f32(K.expand(Q, R, 3, 3)), ref_poses=f32(torch.stack(ref_poses)), que_Ks=f32(K.expand(Q, 3, 3)),
                que_poses=f32(torch.stack(que_poses)), sn=sn, img_h=img_h, img_w=img_w)


def volume_fill(ops, pr):
    c = lambda k: pr[k].cuda()
    mean_in, stdv = ops.ref_volume_fill(c('ref_feats'), c('que_feats'), c('ref_Ks'), c('ref_poses'), c('que_Ks'), c('que_poses'),
                                        pr['sn'], pr['img_h'], pr['img_w'])
    torch.cuda.synchronize()
    Q, Cc = pr['que_feats'].shape[0], pr['que_feats'].shape[-1]
    mean_in = mean_in.cpu().reshape(Q, -1, 2 * Cc)
    return mean_in[..., :Cc], mean_in[..., Cc:], stdv.cpu().reshape(Q, -1, Cc)


def volume_reference(pr):
    """float64 oracle: the grid from the fp32 linspace (as the reference builds it), rotated, projected, sampled."""
    d = lambda k: pr[k].double()
    coords = O.ref_volume_coords(d('que_poses'), pr['sn'])                                   # Q, sn^3, 3
    ref_proj = d('ref_Ks') @ d('ref_poses')
    que_proj = d('que_Ks') @ d('que_poses')
    means, stds, vins = [], [], []
    for qi in range(coords.shape[0]):
        rf = d('ref_feats')[qi].permute(0, 3, 1, 2)                                          # R, C, fh, fw
        v = O.ref_sample_volume(rf, coords[qi:qi + 1].expand(rf.shape[0], -1, -1), ref_proj[qi], pr['img_h'], pr['img_w'])
        means.append(v.mean(0).T)
        stds.append(v.std(0).T)                                                              # unbiased, refiner.py:237
        qf = d('que_feats')[qi:qi + 1].permute(0, 3, 1, 2)
        vins.append(O.ref_sample_volume(qf, coords[qi:qi + 1], que_proj[qi:qi + 1], pr['img_h'], pr['img_w'])[0].T)
    return torch.stack(means), torch.stack(vins), torch.stack(stds)


def volume_atol(pr):
    """The kernel projects in fp32.  A pixel coordinate px = sum of <= 4 terms |K P v| <= ~1350 (f = 100, c <= 64,
    |t| <= 3, |v| <= sqrt 3) through <= 8 roundings, divided by a depth >= 1.27 wherever a voxel lands within a tap of
    the map, puts the fp32 sample point within 8 * 1350 * 2^-24 / 1.27 * 2 ~ 1e-3 image pixels = 2.5e-4 feature
    pixels (maps are 1/4 of the image) of the fp64 one in x and in y.  Bilinear sampling moves by at most the largest
    neighbouring-pixel difference kappa of the zero-padded maps per pixel, so |d sample| <= 2 * 2.5e-4 * kappa; the
    four-tap blend adds 8 roundings of values <= max|f|."""
    maps = torch.cat([pr['ref_feats'].flatten(0, 1), pr['que_feats']], 0).double()
    padded = F.pad(maps.permute(0, 3, 1, 2), (1, 1, 1, 1))
    kappa = max(float((padded[..., 1:, :] - padded[..., :-1, :]).abs().max()),
                float((padded[..., :, 1:] - padded[..., :, :-1]).abs().max()))
    return 2 * 2.5e-4 * kappa + 8 * U * float(maps.abs().max())


VOLUME_CASES = [
    # R, C, sn, Q, size: R != 6 runs ref_volume_fill_kernel<0>; R = 6 runs the C = 128 kernel or, for other C, <6>
    (2, 128, 2, 1, SQUARE), (2, 128, 9, 3, WIDE), (2, 128, 33, 1, WIDE),
    (3, 128, 3, 3, SQUARE), (3, 128, 32, 1, WIDE),
    (5, 128, 9, 1, WIDE), (5, 128, 33, 1, SQUARE),
    (6, 128, 2, 3, WIDE), (6, 128, 32, 3, SQUARE), (6, 128, 33, 1, WIDE), (6, 128, 9, 1, SQUARE),
    (7, 128, 3, 1, WIDE), (7, 128, 32, 1, SQUARE), (7, 128, 9, 3, SQUARE),
    (6, 256, 9, 3, WIDE), (6, 256, 33, 1, SQUARE),
    (6, 64, 9, 1, WIDE), (6, 64, 32, 3, SQUARE),
    (3, 4, 33, 3, WIDE), (3, 4, 2, 1, SQUARE),
    (3, 132, 9, 3, SQUARE), (3, 132, 32, 1, WIDE),
]


@pytest.mark.parametrize('R,Cc,sn,Q,size', VOLUME_CASES)
def test_ref_volume_fill_matches_fp64(ops, R, Cc, sn, Q, size):
    pr = volume_problem(Q, R, Cc, sn, size, seed=1000 * R + 10 * sn + Cc)
    got_mean, got_in, got_std = volume_fill(ops, pr)
    want_mean, want_in, want_std = volume_reference(pr)
    atol = volume_atol(pr)
    rtol = 8 * U                      # the blend, the mean's R adds and the two-pass variance, each a few roundings
    check(f'mean R={R} C={Cc} sn={sn}', got_mean, want_mean, atol, rtol)
    check(f'query sample R={R} C={Cc} sn={sn}', got_in, want_in, atol, rtol)
    # the unbiased std is sqrt(R/(R-1))-Lipschitz in the max-norm of the R samples; with R = 2 the biased one is off by
    # sqrt 2, far outside this
    check(f'std R={R} C={Cc} sn={sn}', got_std, want_std, atol * math.sqrt(R / (R - 1)), rtol)
    # the geometry reaches what it is meant to: zero padding (all taps off) and non-trivial samples
    assert bool((want_in.abs() > 0.1).any())
    if R == 2:
        biased = want_std / math.sqrt(2)
        assert float((got_std.double() - biased).abs().max()) > 10 * atol


@pytest.mark.parametrize('R,c_small,c_big', [(6, 128, 256), (3, 128, 256), (3, 128, 132), (6, 64, 256)])
def test_ref_volume_fill_channel_block_is_bit_identical(ops, R, c_small, c_big):
    """Channels [0, c_small) of a c_big call with features [f, g] are, bit for bit, the c_small call with f: a channel's
    arithmetic does not depend on how many channels follow it.  (6, 128, 256) compares the C = 128 kernel with the
    generic kernel at R = 6, whose comment promises the same arithmetic."""
    pr = volume_problem(3, R, c_big, 17, WIDE, seed=77 + R)
    small = dict(pr, ref_feats=pr['ref_feats'][..., :c_small].contiguous(), que_feats=pr['que_feats'][..., :c_small].contiguous())
    big = volume_fill(ops, pr)
    ref = volume_fill(ops, small)
    for name, b, s in zip(('mean', 'query sample', 'std'), big, ref):
        gap = ulp_gap(b[..., :c_small], s)
        print(f'R={R} C={c_big} vs C={c_small} {name}: max gap {gap} ulp')
        assert gap == 0, f'{name}: channels [0, {c_small}) differ by up to {gap} ulp between C={c_big} and C={c_small}'


# ----------------------------------------------------------------------------------------------------------------------
# g6d_det_score_fuse
# ----------------------------------------------------------------------------------------------------------------------
FRAME = (270, 480)                                        # hs x ws = 33 x 60
SCALES = [-1.0, -0.5, 0.0, 0.5, 1.0, -1.5]               # level-0 rows 20, 24, 36, 48, 68, 12 around hs = 33
STATS = O.DET_DEFAULT_CFG['vgg_score_stats']
CLIP = float(O.DET_DEFAULT_CFG['vgg_score_max'])


def fuse_problem(n_scales, rfn, qn, seed):
    g = gen(seed)
    hq, wq = FRAME
    raw = []        # raw[s][l]: [qn, H/2^l, W/2^l, rfn] fp32, raw correlation values straddling mu +- clip * sigma
    for ht, wt in O.det_scale_sizes(hq, wq, SCALES[:n_scales]):
        raw.append([STATS[l][0] + STATS[l][1] * CLIP * 0.8 * torch.randn(qn, ht // 8 >> l, wt // 8 >> l, rfn, generator=g)
                    for l in range(3)])
    nin = 3 * n_scales
    w = dict(w1=torch.randn(64, nin, generator=g) / math.sqrt(nin), b1=0.5 * torch.randn(64, generator=g),
             w2=torch.randn(64, 64, generator=g) / 8, b2=0.5 * torch.randn(64, generator=g))
    return raw, w


def score_fuse(ops, raw, w, rfn, qn):
    hs, ws = FRAME[0] // 8, FRAME[1] // 8
    maps = [[t.cuda() for t in lv] for lv in raw]
    sizes = [[(t.shape[1], t.shape[2]) for t in lv] for lv in raw]
    c = {k: v.cuda() for k, v in w.items()}
    out = ops.det_score_fuse(maps, sizes, rfn, hs, ws, STATS, CLIP, c['w1'], c['b1'], c['w2'], c['b2'], qn)
    return out.cpu()


def score_fuse_reference(raw, w, chunk=33):
    """oracle.det_fuse_scores in float64, over references in chunks of `chunk` (the max over references is exact, so
    the max of the chunks' maxima is the same number) to bound the memory of score_conv's [qn, 64, rfn, hs, ws]."""
    hs, ws = FRAME[0] // 8, FRAME[1] // 8
    n_scales = len(raw)
    sd = {'score_conv.0.weight': w['w1'].double().reshape(64, 3 * n_scales, 1, 1, 1), 'score_conv.0.bias': w['b1'].double(),
          'score_conv.2.weight': w['w2'].double().reshape(64, 64, 1, 1, 1), 'score_conv.2.bias': w['b2'].double()}
    cfg = {'vgg_score_stats': STATS, 'vgg_score_max': CLIP}
    rfn = raw[0][0].shape[-1]
    out = None
    for r0 in range(0, rfn, chunk):
        sub = [[t[..., r0:r0 + chunk].permute(0, 3, 1, 2).double() for t in lv] for lv in raw]
        feats, _ = O.det_fuse_scores(sd, cfg, sub, hs, ws)
        out = feats if out is None else torch.maximum(out, feats)
    return out.permute(0, 2, 3, 1)                                                            # qn, hs, ws, 64


def score_fuse_atol(raw, w):
    """A forward error bound.  Inputs: the fp32 bilinear source coordinate (scale * (dst + 0.5) - 0.5, scale = Hc / hs)
    is within 4 roundings of the level-0 size of the fp64 one, moving the blend by that times the <= 2 clip jump between
    taps; normalising (fp32 1/sigma) and blending add ~8 roundings of values <= clip.  Hidden: the
    input error through sum_i |w1| plus (3S + 1) roundings of a sum bounded by |b1| + sum_i |w1| clip.  Output: the
    hidden error through sum_h |w2| plus 65 roundings of a sum bounded by |b2| + sum_h |w2| max hidden."""
    hmax = max(max(lv[0].shape[1], lv[0].shape[2]) for lv in raw)
    e_in = 4 * U * hmax * 2 * CLIP + 8 * U * CLIP
    w1, b1, w2, b2 = (w[k].double() for k in ('w1', 'b1', 'w2', 'b2'))
    hid_bound = b1.abs() + w1.abs().sum(1) * CLIP
    e_hid = w1.abs().sum(1) * e_in + (w1.shape[1] + 1) * U * hid_bound
    out_bound = b2.abs() + w2.abs() @ hid_bound
    return float((w2.abs() @ e_hid + 65 * U * out_bound).max())


FUSE_CASES = [   # n_scales, rfn, qn: every instantiation, one and several 64-reference chunks, partial last chunks
    (1, 1, 1), (1, 65, 3), (2, 3, 3), (2, 130, 1), (3, 33, 1), (3, 64, 3),
    (4, 64, 1), (4, 130, 1), (5, 65, 1), (5, 1, 3), (6, 130, 1), (6, 3, 3),
]


@pytest.mark.parametrize('n_scales,rfn,qn', FUSE_CASES)
def test_det_score_fuse_matches_fp64(ops, n_scales, rfn, qn):
    raw, w = fuse_problem(n_scales, rfn, qn, seed=100 * n_scales + rfn + qn)
    clipped = sum(float(((t - STATS[l][0]).abs() > CLIP * STATS[l][1]).double().mean()) for lv in raw for l, t in enumerate(lv))
    assert clipped > 0.05 * 3 * n_scales, 'the raw values should often lie beyond the clip'
    got = score_fuse(ops, raw, w, rfn, qn)
    want = score_fuse_reference(raw, w)
    check(f'score fuse S={n_scales} rfn={rfn} qn={qn}', got, want, score_fuse_atol(raw, w), 0.0)


@pytest.mark.parametrize('n_scales', [2, 6])
def test_det_score_fuse_chunks_are_bit_identical(ops, n_scales):
    """rfn = 130 runs three 64-reference chunks, the later ones merged by the read-modify-write fmaxf: bit for bit the
    elementwise max of the calls on references [0, 64), [64, 128) and [128, 130), whose per-reference arithmetic is
    the same whichever lane computes it."""
    rfn, qn = 130, 2
    raw, w = fuse_problem(n_scales, rfn, qn, seed=9 + n_scales)
    full = score_fuse(ops, raw, w, rfn, qn)
    parts = []
    for r0, r1 in ((0, 64), (64, 128), (128, 130)):
        sub = [[t[..., r0:r1].contiguous() for t in lv] for lv in raw]
        parts.append(score_fuse(ops, sub, w, r1 - r0, qn))
    want = torch.maximum(torch.maximum(parts[0], parts[1]), parts[2])
    gap = ulp_gap(full, want)
    print(f'score fuse S={n_scales} rfn=130 vs max of the chunks: max gap {gap} ulp')
    assert gap == 0
    # every chunk wins somewhere: the merge is exercised in both directions
    for p in parts:
        assert bool((p == full).any())


# ----------------------------------------------------------------------------------------------------------------------
# selector tail: g6d_sel_vp_norm, g6d_sel_max_angle_add, g6d_sel_parse
# ----------------------------------------------------------------------------------------------------------------------
SENTINEL = -7777.0


@pytest.mark.parametrize('cstride,coff', [(516, 512), (4, 0)])
@pytest.mark.parametrize('L', [1, 3])
@pytest.mark.parametrize('n', [1, 7, 320, 5000])
def test_sel_vp_norm_matches_fp64(ops, L, n, cstride, coff):
    eps = 1e-5
    score = 1000.0 + torch.randn(L, n, generator=gen(n + L))            # large mean, unit spread
    feats = torch.full((n, cstride), SENTINEL).cuda()
    ops.sel_vp_norm(score.cuda(), feats, coff, eps)
    got = feats.cpu()
    s = score.double()
    want = (s - s.mean(1, keepdim=True)) / torch.sqrt(s.var(1, unbiased=False, keepdim=True) + eps)
    # the kernel subtracts the fp32-rounded mean, <= half an ulp of |mean| ~ 1e3 (2^-15) off, and rounds the difference
    # and the product by rstd: 2^-14 * rstd covers the three
    rstd = 1 / torch.sqrt(s.var(1, unbiased=False, keepdim=True) + eps)
    atol = 2.0 ** -14 * rstd.T
    check(f'vp_norm L={L} n={n} coff={coff}', got[:, coff:coff + L], want.T, atol, 4 * U)
    assert bool((got[:, :coff] == SENTINEL).all()), 'channels before coff must be left alone'
    assert bool((got[:, coff + L:] == 0).all()), 'the padding channels after the scores must be cleared'


@pytest.mark.parametrize('an', [1, 5])
@pytest.mark.parametrize('rfn', [1, 64])
@pytest.mark.parametrize('Cc', [512, 7])
def test_sel_max_angle_add_bit_exact(ops, rfn, an, Cc):
    g = gen(rfn * an + Cc)
    x = torch.randn(rfn, an, Cc, generator=g) * 3
    embed = torch.randn(rfn, Cc, generator=g)
    got = ops.sel_max_angle_add(x.cuda(), embed.cuda()).cpu()
    want = torch.max(x, 1)[0] + embed
    print(f'max_angle_add rfn={rfn} an={an} C={Cc}: max gap {ulp_gap(got, want)} ulp')
    assert torch.equal(got, want)


def _parse_rows(rfn, g):
    nan, inf = float('nan'), float('inf')
    rows = []
    r = torch.randn(rfn, generator=g)
    rows.append(r.clone())                                           # plain
    t = r.clone()
    t[rfn // 3] = t[2 * rfn // 3] = t[-1] = float(r.max()) + 1       # a three-way tie: the first wins
    rows.append(t)
    t = r.clone()
    t[0] = nan                                                       # a leading NaN is the maximum
    rows.append(t)
    if rfn >= 3:
        t = r.clone()
        t[1] = float(r.max()) + 5
        t[rfn // 2] = nan
        t[-1] = nan                                                  # a later NaN beats a larger finite value; the first NaN wins
        rows.append(t)
    rows.append(torch.full((rfn,), -inf))                            # all -inf: index 0
    t = r.clone()
    t[-1] = inf                                                      # +inf at the end
    rows.append(t)
    return torch.stack(rows)


@pytest.mark.parametrize('rfn', [1, 2, 1000])
def test_sel_parse_matches_torch_argmax(ops, rfn):
    g = gen(rfn)
    logits = _parse_rows(rfn, g)
    angles = torch.randn(logits.shape, generator=g)
    idx, out = ops.sel_parse(logits.cuda(), angles.cuda())
    idx, out = idx.cpu(), out.cpu()
    want_idx = torch.argmax(logits, 1)                               # selector.py:172
    assert torch.equal(idx, want_idx), (idx.tolist(), want_idx.tolist())
    ar = torch.arange(logits.shape[0])
    assert torch.equal(out[:, 0], angles[ar, want_idx])
    assert torch.equal(out[:, 1].isnan(), logits[ar, want_idx].isnan())
    fin = ~out[:, 1].isnan()
    assert torch.equal(out[fin, 1], logits[ar, want_idx][fin])


# ----------------------------------------------------------------------------------------------------------------------
# g6d_avgpool_affine
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('spatial', [1, 16, 49])
@pytest.mark.parametrize('Cc', [3, 512])
@pytest.mark.parametrize('affine', [False, True])
@pytest.mark.parametrize('act', ['none', 'relu'])
def test_avgpool_affine_matches_fp64(ops, spatial, Cc, affine, act):
    """mean over `spatial` rows of act(x * scale[g] + shift[g]), group g = row // rows_per_group; rows_per_group =
    2 * spatial + 1 makes a group boundary fall inside a pooling window.  ReLU acts on each row before the mean."""
    g = gen(spatial * 7 + Cc + affine)
    n_out = 6
    rows = n_out * spatial
    rpg = 2 * spatial + 1
    groups = (rows + rpg - 1) // rpg
    x = torch.randn(rows, Cc, generator=g)
    scale = shift = None
    v = x.double()
    if affine:
        scale = 1 + 0.5 * torch.randn(groups, Cc, generator=g)
        shift = 0.5 * torch.randn(groups, Cc, generator=g)
        gi = torch.arange(rows) // rpg
        v = v * scale.double()[gi] + shift.double()[gi]
    a = ops.ACT_RELU if act == 'relu' else ops.ACT_NONE
    if act == 'relu':
        v = v.clamp_min(0)
    want = v.reshape(n_out, spatial, Cc).mean(1)
    got = ops.avgpool_affine(x.cuda(), spatial, None if scale is None else scale.cuda(), None if shift is None else shift.cuda(),
                             rows_per_group=rpg, act=a)
    # one fma per row, `spatial` sequential adds, one division: spatial + 2 roundings of values <= max|v|
    check(f'avgpool spatial={spatial} C={Cc} affine={affine} act={act}', got, want, (spatial + 2) * U * float(v.abs().max()), 2 * U)


# ----------------------------------------------------------------------------------------------------------------------
# g6d_ref_pose_heads
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [1, 31, 512, 1000])
@pytest.mark.parametrize('M', [1, 9, 200])
def test_ref_pose_heads_matches_fp64(ops, M, K):
    g = gen(M * 1000 + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(7, K, generator=g) / math.sqrt(K)
    b = torch.randn(7, generator=g)
    b[:4] = 0
    x[0] = 0                                                        # row 0: a zero quaternion, F.normalize's eps clamp
    got = ops.ref_pose_heads(x.cuda(), w.cuda(), b.cuda()).cpu()
    res = x.double() @ w.double().T + b.double()
    want = torch.cat([F.normalize(res[:, :4], dim=1), res[:, 4:]], 1)
    # each lane sums ceil(K/32) products in sequence, a 5-level warp tree and the bias follow: gamma_d * sum |x w| + |b|
    d = -(-K // 32) + 6
    e = d * U * (x.double().abs() @ w.double().abs().T + b.double().abs())                  # M, 7
    # normalising q = r / |r| turns an error e_r into <= 2 |e_r| / |r| plus a few roundings of |q| <= 1
    nrm = res[:, :4].norm(dim=1, keepdim=True)
    eq = torch.where(nrm > 0, 2 * e[:, :4].norm(dim=1, keepdim=True) / nrm, torch.zeros_like(nrm)) + 6 * U
    check(f'pose heads M={M} K={K}', got, want, torch.cat([eq.expand(-1, 4), e[:, 4:]], 1), 0.0)
    assert bool((got[0, :4] == 0).all()), 'a zero quaternion normalises to zero (eps clamp), not NaN'
