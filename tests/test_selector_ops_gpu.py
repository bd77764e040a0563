"""The selector's streaming kernels (the correlation score at one and at three pyramid levels, the reference
sums and the closed-form first InstanceNorm of the correlation volume) and its attention and LayerNorm on
the GPU, against float64 CPU restatements of the same operations, at every instantiation and at the shapes
where indexing goes wrong: row pairs that straddle a level boundary, CTA chunks that cover many small items
and items shared by several CTAs, slice loops of several trips, channel counts that are not a multiple of
32, key counts on either side of the 48 KB shared-memory line.

A tolerance here is |got - want| <= atol + rtol*|want|, each stated with the fp32 operation count and data
magnitude it comes from; every check prints the worst error it saw and its fraction of the tolerance.
Where two kernel paths do the same fp32 arithmetic the check is bit for bit."""
import math

import pytest
import torch
import torch.nn.functional as F

from test_tail_ops_gpu import U, check, gen, ulp_gap

pytestmark = pytest.mark.gpu

C512 = 512


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


# ----------------------------------------------------------------------------------------------------------------------
# g6d_sel_corr_score3 / g6d_sel_corr_score
# ----------------------------------------------------------------------------------------------------------------------
def level_problem(S, Ps, seed, Cc=C512):
    """refs[l] [S, P_l, C] and qs[l] [P_l, C], uniform in [0, 1), with every third slice negated so that all its inner
    products, and so its max, are negative.  The three levels are consecutive views of ONE buffer (likewise the
    queries), as in a packed reference record: an index that runs past the end of a level reads the next level's
    data, a wrong number rather than an out-of-bounds access."""
    g = gen(seed)
    n_ref = sum(S * P * Cc for P in Ps)
    flat = torch.rand(n_ref, generator=g)
    qflat = torch.rand(sum(P * Cc for P in Ps), generator=g)
    refs, qs, o, oq = [], [], 0, 0
    for P in Ps:
        r = flat[o:o + S * P * Cc].view(S, P, Cc)
        r[1::3] *= -1
        refs.append(r)
        qs.append(qflat[oq:oq + P * Cc].view(P, Cc))
        o += S * P * Cc
        oq += P * Cc
    return flat, qflat, refs, qs


def to_device(flat, qflat, refs, qs):
    """The same views over one device buffer each."""
    fd, qd = flat.cuda(), qflat.cuda()
    out_r, out_q, o, oq = [], [], 0, 0
    for r, q in zip(refs, qs):
        out_r.append(fd[o:o + r.numel()].view(r.shape))
        out_q.append(qd[oq:oq + q.numel()].view(q.shape))
        o += r.numel()
        oq += q.numel()
    return out_r, out_q


def dots64(ref, q, chunk=64):
    """t[s, p] = sum_c q[p, c] ref[s, p, c] and sum_c |q ref| in float64, a few slices at a time."""
    t, a = [], []
    qd = q.double()
    for s0 in range(0, ref.shape[0], chunk):
        r = ref[s0:s0 + chunk].double()
        t.append(torch.einsum('spc,pc->sp', r, qd))
        a.append(torch.einsum('spc,pc->sp', r.abs(), qd.abs()))
    return torch.cat(t), torch.cat(a)


def score_reference(t, a, dot_depth, sum_depth):
    """score[s] = sum_p t (t / max_p t) in float64, and its forward error bound.  Each t carries the error of a
    dot_depth-deep fp32 chain, e_p = dot_depth u sum_c |q r|; the max moves by at most max_p e_p.  To first order the
    score moves by sum_p (2 |t_p| e_p + t_p^2 max e / |m|) / |m|; then t / m and t * (t / m) round once each and the
    P terms, all of the sign of m, are summed sum_depth deep."""
    m = t.max(1, keepdim=True)[0]
    want = torch.sum(t * (t / m), 1)
    e = dot_depth * U * a
    E = e.max(1, keepdim=True)[0]
    tm = t.abs() / m.abs()
    bound = torch.sum(2 * tm * e + tm * tm * E, 1) + (sum_depth + 2) * U * torch.sum(t * tm, 1).abs()
    return want, bound


PSETS = [(256, 64, 16), (25, 9, 4), (1, 1, 1), (3, 5, 7)]
SCORE3_CASES = [(S, Ps) for Ps in PSETS for S in (1, 2, 7, 320)] + [(641, (256, 64, 16))]


@pytest.mark.parametrize('S,Ps', SCORE3_CASES)
def test_sel_corr_score3_matches_fp64(ops, S, Ps):
    """Fused (one launch, completion counters) and unfused (dots + finish) against float64.  With S * P_l odd a row pair
    straddles a level boundary; small P puts many items into one CTA's chunk, large S * P_0 spreads an item over
    several CTAs.  The two paths do the same fp32 arithmetic, so they agree bit for bit."""
    flat, qflat, refs, qs = level_problem(S, Ps, seed=S * 1000 + sum(Ps))
    dr, dq = to_device(flat, qflat, refs, qs)
    counters = torch.zeros(3 * S, dtype=torch.int32, device='cuda')
    fused = ops.sel_corr_score3(dr, dq, counters=counters)
    assert int(counters.abs().sum()) == 0, 'the completing CTA leaves every counter zero'
    unfused = ops.sel_corr_score3(dr, dq)
    fused, unfused = fused.cpu(), unfused.cpu()
    assert torch.equal(fused, unfused), f'fused and unfused differ by up to {ulp_gap(fused, unfused)} ulp'
    for l, P in enumerate(Ps):
        t, a = dots64(refs[l], qs[l])
        # 16 sequential fmas per lane (4 float4) and a 5-level shuffle tree per dot; ceil(P/32) sequential adds per lane
        # and a 5-level tree for the score
        want, bound = score_reference(t, a, 16 + 5, -(-P // 32) + 5)
        check(f'score3 S={S} P={Ps} level {l}', fused[l], want, bound, 0.0)
        if S >= 2:
            assert bool((want[1::3] < 0).all()) and bool((want[0::3] > 0).all()), 'a negative max gives a negative score'


def test_sel_corr_score3_alternating_records(ops):
    """Two reference records of different sizes, each with its own counters, used alternately: every call gives what
    that record gives alone (the counters carry nothing from one call to the next)."""
    recs = []
    for S, Ps, seed in ((7, (25, 9, 4), 5), (320, (3, 5, 7), 6)):
        flat, qflat, refs, qs = level_problem(S, Ps, seed)
        dr, dq = to_device(flat, qflat, refs, qs)
        counters = torch.zeros(3 * S, dtype=torch.int32, device='cuda')
        recs.append((dr, dq, counters, ops.sel_corr_score3(dr, dq, counters=counters).cpu()))
    for _ in range(3):
        for dr, dq, counters, alone in recs:
            got = ops.sel_corr_score3(dr, dq, counters=counters).cpu()
            assert torch.equal(got, alone)
            assert int(counters.abs().sum()) == 0


SCORE_CASES = [(Cc, P, S) for Cc in (128, 256, 512) for P, S in ((1, 1100), (7, 1100), (256, 13), (8192, 2))]


@pytest.mark.parametrize('Cc,P,S', SCORE_CASES)
def test_sel_corr_score_matches_fp64(ops, Cc, P, S):
    """Every channel instantiation; S = 1100 > 8 * 132 slices makes each CTA's slice loop run more than once."""
    flat, qflat, refs, qs = level_problem(S, (P,), seed=Cc + P + S, Cc=Cc)
    dr, dq = to_device(flat, qflat, refs, qs)
    got = ops.sel_corr_score(dr[0], dq[0]).cpu()
    t, a = dots64(refs[0], qs[0])
    # C/128 float4 per lane: C/32 sequential fmas and a 5-level tree per dot; the score sums ceil(P/256) terms per
    # thread, a 5-level tree and 8 warps in sequence
    want, bound = score_reference(t, a, Cc // 32 + 5, -(-P // 256) + 12)
    check(f'score C={Cc} P={P} S={S}', got, want, bound, 0.0)


@pytest.mark.parametrize('P', [1, 7, 256])
def test_sel_corr_score_agrees_with_score3(ops, P):
    """At C = 512 both kernels compute every inner product with the same lane-wise fma chain and shuffle tree, so the
    terms t (t / m) are the same numbers; only the order of the P-term sum differs (ceil(P/256) + 5 + 7 deep against
    ceil(P/32) + 5).  The terms share one sign, so each sum is within depth * u * |score| of the exact one and the two
    differ by fewer than d1 + d2 ulp of the score."""
    S = 41
    flat, qflat, refs, qs = level_problem(S, (P, P, P), seed=P)
    dr, dq = to_device(flat, qflat, refs, qs)
    three = ops.sel_corr_score3(dr, dq, counters=torch.zeros(3 * S, dtype=torch.int32, device='cuda')).cpu()
    limit = (-(-P // 256) + 12) + (-(-P // 32) + 5)
    for l in range(3):
        one = ops.sel_corr_score(dr[l], dq[l]).cpu()
        gap = ulp_gap(one, three[l])
        print(f'score vs score3 P={P} level {l}: max gap {gap} ulp (bound {limit})')
        assert gap < limit
        if P == 1:
            assert gap == 0, 'one term: nothing to reorder'


# ----------------------------------------------------------------------------------------------------------------------
# g6d_sel_ref_sums, g6d_sel_corr_prologue
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S', [1, 15, 16, 17, 320, 1000])
def test_sel_ref_sums_matches_fp64(ops, S):
    """16 slices per block along grid.y, blocks merged by fp64 atomics in no fixed order: a tolerance, not bits.  Every
    sum is of fp32 values (exact in fp64) through at most S fp64 additions: S 2^-53 sum |v|."""
    P, Cc = 16, 512
    ref = torch.randn(S, P, Cc, generator=gen(S)) * 3 + 1
    s1, s2 = ops.sel_ref_sums(ref.cuda())
    r = ref.double()
    check(f'ref sums S={S} sum', s1.cpu(), r.sum(0), S * 2.0 ** -53 * r.abs().sum(0), 0.0)
    check(f'ref sums S={S} sum of squares', s2.cpu(), (r * r).sum(0), (S + 1) * 2.0 ** -53 * (r * r).sum(0), 0.0)


def prologue_problem(S, P, Cc, seed):
    """ref in [-0.5, 1.5) and q in [0.5, 1.5): the volume q * ref has mean ~ its spread, like the normalised features."""
    g = gen(seed)
    ref = torch.rand(S, P, Cc, generator=g) * 2 - 0.5
    q = torch.rand(P, Cc, generator=g) + 0.5
    return ref, q


PROLOGUE_CASES = [(12, 16, 512), (12, 64, 512), (5, 256, 512), (7, 9, 4), (7, 9, 33), (3, 20, 100)]


@pytest.mark.parametrize('S,P,Cc', PROLOGUE_CASES)
def test_sel_corr_prologue_matches_fp64(ops, S, P, Cc):
    """The closed form: mean_c = sum_p q A / N, E2_c = sum_p q^2 B / N over N = S P, var = E2 - mean^2, then
    scale = q rstd (fp32) and shift = -mean rstd.  Then end to end: ref * scale + shift, what the PRO_CORR loader
    computes, equals float64 F.instance_norm of the explicit volume q[p, c] ref[s, p, c] over (S, P) -- the operation
    the reference runs first on the correlation volume."""
    eps = 1e-5
    ref, q = prologue_problem(S, P, Cc, seed=S * P + Cc)
    s1, s2 = ops.sel_ref_sums(ref.cuda())
    scale, shift = ops.sel_corr_prologue(q.cuda(), s1, s2, S, eps)
    scale, shift = scale.cpu(), shift.cpu()
    vol = q.double()[None] * ref.double()                                            # S, P, C
    mean = vol.mean((0, 1))
    var = vol.var((0, 1), unbiased=False)
    rstd = 1 / torch.sqrt(var + eps)
    # float64 sums of N products through ~S + P + 8 roundings, then E2 - mean^2 cancels: the variance is within
    # d = (S + P + 8) 2^-52 (E2 + mean^2); rstd moves by d / (2 (var + eps)) relative; the casts to fp32 and the fp32
    # product q * rstd add 2 roundings
    e2 = (vol * vol).mean((0, 1))
    rel = (S + P + 8) * 2.0 ** -52 * (e2 + mean * mean) / (2 * (var + eps)) + 2 * U
    check(f'prologue S={S} P={P} C={Cc} shift', shift, -mean * rstd, rel * (mean * rstd).abs(), 0.0)
    check(f'prologue S={S} P={P} C={Cc} scale', scale, q.double() * rstd, rel * (q.double() * rstd), 0.0)
    # end to end against the explicit InstanceNorm (biased variance over the S*P positions of each channel)
    x = vol.permute(2, 0, 1).reshape(1, Cc, S * P)
    norm = F.instance_norm(x, eps=eps).reshape(Cc, S, P).permute(1, 2, 0)
    got = ref.double() * scale.double()[None] + shift.double()
    # the loader's fma adds one rounding of |ref scale| + |shift|; scale and shift carry rel each
    atol = (rel + U) * ((ref.double() * scale.double()[None]).abs() + shift.double().abs())
    check(f'prologue S={S} P={P} C={Cc} ref*scale+shift vs instance_norm', got, norm, atol, 0.0)


# ----------------------------------------------------------------------------------------------------------------------
# g6d_attention_headmajor, g6d_attention
# ----------------------------------------------------------------------------------------------------------------------
LOGIT_MAX = 90.0      # beyond log(FLT_MAX) = 88.7: without the max subtraction exp overflows to inf


def attention_problem(n, Cc, heads, seed):
    """q, k, v in the reference's channel order (c = d*heads + h).  Keys and queries share a random direction per
    head, so the logits q.k / sqrt(D) spread over about +-LOGIT_MAX and the softmax has a few dominant keys."""
    g = gen(seed)
    D = Cc // heads
    q = torch.randn(n, D, heads, generator=g)
    k = torch.randn(n, D, heads, generator=g)
    dirn = F.normalize(torch.randn(1, D, heads, generator=g), dim=1)
    amp_q = torch.randn(n, 1, heads, generator=g)
    amp_k = torch.randn(n, 1, heads, generator=g)
    q = q * 0.3 + amp_q * dirn * 3
    k = k * 0.3 + amp_k * dirn * 3
    # scale q per head so that the largest |logit| of every head is LOGIT_MAX
    for h in range(heads):
        lg = float((q[:, :, h].double() @ k[:, :, h].double().T).abs().max())
        q[:, :, h] *= LOGIT_MAX * math.sqrt(D) / lg
    v =torch.randn(n, D, heads, generator=g)
    return q.reshape(n, Cc), k.reshape(n, Cc), v.reshape(n, Cc)


def attention_reference(q, k, v, heads):
    """float64 softmax(q_h k_h^T / sqrt(D)) v_h per head (attention.py:4-17), and a forward error bound per element.
    A logit is a D-term fp32 dot (D + 5 roundings with the scaling by an rsqrtf): |dl| <= (D + 5) u sum_d |q k| /
    sqrt(D); the subtraction of the row maximum rounds once more, u |l - max l| <= 2 u max|l|.  Perturbing the logits by at most dl moves the softmax average of v by at most 2 dl max|v|; expf (2 ulp),
    the n-term sum of the weights and the n-term weighted value sum add (2 n + 8) u max|v|."""
    n, Cc = q.shape
    D = Cc // heads
    qd, kd, vd = (t.double().reshape(n, D, heads) for t in (q, k, v))
    out = torch.empty(n, D, heads, dtype=torch.float64)
    atol = torch.empty(n, D, heads, dtype=torch.float64)
    for h in range(heads):
        lg = qd[:, :, h] @ kd[:, :, h].T / math.sqrt(D)
        out[:, :, h] = torch.softmax(lg, 1) @ vd[:, :, h]
        dl = (D + 5) * U * float((qd[:, :, h].abs() @ kd[:, :, h].abs().T).max()) / math.sqrt(D) + 2 * U * float(lg.abs().max())
        vmax = float(vd[:, :, h].abs().max())
        atol[:, :, h] = 2 * dl * vmax + (2 * n + 8) * U * vmax
        if n > 1:
            assert float(lg.abs().max()) > 88.8, 'the logits reach beyond exp\'s fp32 range'
    return out.reshape(n, Cc), atol.reshape(n, Cc)


def head_major(t, heads):
    """reference channel order c = d*heads + h -> head-major c' = h*D + d"""
    n, Cc = t.shape
    return t.reshape(n, Cc // heads, heads).permute(0, 2, 1).reshape(n, Cc).contiguous()


HM_CASES = [(n, heads) for n in (1, 7, 8, 31, 33, 320, 1184, 1185) for heads in (1, 2, 8)] + [(2048, 8)]


@pytest.mark.parametrize('n,heads', HM_CASES)
def test_attention_headmajor_matches_fp64(ops, n, heads):
    """The tiled kernel at every key-tile remainder; n = 1184 keeps the score rows within 48 KB of shared memory,
    1185 and 2048 need the opted-in 96 KB."""
    Cc = 64 * heads
    q, k, v = attention_problem(n, Cc, heads, seed=n * 10 + heads)
    want, atol = attention_reference(q, k, v, heads)
    got = ops.attention(*(head_major(t, heads).cuda() for t in (q, k, v)), heads, head_major=True).cpu()
    check(f'attention head-major n={n} heads={heads}', got, head_major(want, heads), head_major(atol, heads), 0.0)
    assert bool(torch.isfinite(got).all())


REF_CASES = [(1, 512, 8), (24, 512, 8), (333, 512, 16), (1000, 512, 1), (2500, 256, 16), (4096, 64, 1)]


@pytest.mark.parametrize('n,Cc,heads', REF_CASES)
def test_attention_reference_order_matches_fp64(ops, n, Cc, heads):
    q, k, v = attention_problem(n, Cc, heads, seed=n + Cc + heads)
    want, atol = attention_reference(q, k, v, heads)
    got = ops.attention(q.cuda(), k.cuda(), v.cuda(), heads).cpu()
    check(f'attention reference order n={n} C={Cc} heads={heads}', got, want, atol, 0.0)


@pytest.mark.parametrize('n', [7, 320])
def test_attention_kernels_agree(ops, n):
    """The two kernels sum in different orders, so not bit for bit: each is within its bound of float64, and so within
    the sum of the two bounds of each other."""
    heads, Cc = 8, 512
    q, k, v = attention_problem(n, Cc, heads, seed=99 + n)
    _, atol = attention_reference(q, k, v, heads)
    a = ops.attention(q.cuda(), k.cuda(), v.cuda(), heads).cpu()
    b = ops.attention(*(head_major(t, heads).cuda() for t in (q, k, v)), heads, head_major=True).cpu()
    check(f'attention kernels n={n}', head_major(a, heads), b, 2 * head_major(atol, heads), 0.0)


# ----------------------------------------------------------------------------------------------------------------------
# g6d_layernorm
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rows', [1, 5, 333])
@pytest.mark.parametrize('Cc', [1, 33, 100, 512, 1024])
def test_layernorm_matches_fp64(ops, Cc, rows):
    """One warp per row, 4 rows per block; data with mean / std = 100.  The kernel's mean is a fp32 sum of C terms,
    ceil(C/32) deep per lane, a 5-level tree and the division: within dm = (ceil(C/32) + 6) u sum|x| / C of the exact
    one.  x - mean then carries dm; the centred sum of squares sum (x - m~)^2 = sum (x - m)^2 + C dm^2 and its own
    ceil(C/32) + 5 roundings give the variance within (ceil(C/32) + 7) u var + dm^2 (+ an fma rounding per term);
    rsqrtf adds 2 ulp.  So out = (x - m~) rstd gamma + beta is within dm rstd |gamma| + |x - m| rstd |gamma| dr +
    3 u (|out - beta| + |beta|), dr the relative rstd error."""
    eps = 1e-5
    g = gen(Cc * 7 + rows)
    x = 100 + torch.randn(rows, Cc, generator=g)
    gam = 1 + 0.5 * torch.randn(Cc, generator=g)
    bet = torch.randn(Cc, generator=g)
    got = ops.layernorm(x.cuda(), gam.cuda(), bet.cuda(), eps).cpu()
    xd = x.double()
    want = F.layer_norm(xd, (Cc,), gam.double(), bet.double(), eps)
    depth = -(-Cc // 32)
    dm = (depth + 6) * U * xd.abs().sum(1, keepdim=True) / Cc
    var = xd.var(1, unbiased=False, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    dr = 0.5 * ((depth + 7) * U * var + dm * dm) / (var + eps) + 3 * U
    cen = (xd - xd.mean(1, keepdim=True)).abs()
    atol = dm * rstd * gam.double().abs() + cen * rstd * gam.double().abs() * dr + 3 * U * ((want - bet.double()).abs() + bet.double().abs())
    check(f'layernorm C={Cc} rows={rows}', got, want, atol, 0.0)
