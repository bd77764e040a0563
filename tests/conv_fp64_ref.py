"""One fp64 reference and one error model for every convolution path of ops.conv.

For a call y = ops.conv(x, pc, prologue, pro_scale, pro_shift, group_rows, act, in_coff, out, out_coff) the reference
is built from the fp32 operands alone, in float64 on the tensors' device:

    x'   = the prologue applied to the in-bounds input elements of channels [in_coff, in_coff + Cin); the zero padding
           stays zero, because the kernels apply the prologue while gathering in-bounds taps only:
             G6D_PRO_AFFINE       x * scale[g, c] + shift[g, c],  g = batch item // group_rows
             G6D_PRO_AFFINE_RELU  the same, then ReLU
             G6D_PRO_CORR         x * scale[p, c] + shift[c],     p = the input pixel's position in its D*H*W plane
    ref  = act(sum_k x'_k w_k + b)
    mag  = sum_k |x'_k w_k| + |b|
    s    = sqrt(sum_k (x'_k w_k)^2)

and the result is checked two ways:

 (a) per element, |y - ref| <= TAU_A * mag.  ReLU and leaky ReLU are 1-Lipschitz, so comparing with act(ref) is
     enough.  A structural error (a wrong or missing tap, K-block, tile, bias, padding element, prologue, channel slice
     or K split) moves an element by about mag / K or more, far above the bound.
 (b) per case, rms over the elements with s > 0 of (y - ref) / s <= TAU_B.  This is the accuracy class: the split
     operands (hi + lo) keep every product fp32-faithful, so the error is the fp32 accumulation's, a few 1e-6 s over
     chains of up to 2048 K terms; dropping the lo half of one operand costs about 2^-12 s.

Same-sign operands (post-ReLU activations against post-ReLU correlation kernels) make the error of a long fp32
accumulation grow with the sum itself instead of with s: measured on the detector's correlation, (b) reaches 7.7e-5,
as much as a dropped lo half would cost with signed data, so there (b) does not separate the classes.  Such a call
(median |ref| / mag above COHERENT) keeps (a); the signed cases of the same kernels carry (b).

The bounds were calibrated on an H100 SXM (80 GB, 700 W power limit) over every case of test_conv_fp64_gpu.py, its
production replay included; the worst measured value is written next to each constant.  Every positive case passes with
at least 4x margin and every negative control of that file fails by at least 8x.

Two forms of the same arithmetic: `reference` runs whole tensors through torch's fp64 convolution; `reference_rows`
gathers the fp64 patches of chosen output rows in chunks (a sampled check of a layer whose full fp64 conv would be
too large, e.g. the detector's correlation with K = 115200).  test_conv_fp64_cpu.py checks both against a direct
per-element loop.
"""
import torch
import torch.nn.functional as F

PRO_NONE, PRO_AFFINE, PRO_AFFINE_RELU, PRO_CORR = 0, 1, 2, 3
ACT_NONE, ACT_RELU, ACT_LEAKY01 = 0, 1, 2
TC_TF32, TC_F16 = 0, 1

# (a) |y - ref| <= TAU_A * mag.  Worst measured: 4.5e-6 (the detector's 1x7 correlation in the production replay: same-sign
# products, 640-term chains), below 6.5e-7 everywhere else.  The changed border pixel of the negative control moves its
# outputs by at least 5.4e-3 mag.
TAU_A = 2.0 ** -15
# (b) rms((y - ref) / s) of the tensor-core path (fp32-faithful split operands).  Worst measured: 1.75e-6 (a 3x3x512
# layer of the production replay), 9.5e-7 over the matrix.  Without the lo half of the weights: 1.49e-4 (fp16 operands,
# BN 128) and 2.06e-4 (tf32).
TAU_B_TC = 1.5e-5
# (b) of the FFMA path (plain fp32 products, fmaf accumulation).  Worst measured: 2.2e-7 (matrix), 1.7e-7 (replay).
TAU_B_FFMA = 2e-6
# a call whose sums are coherent (median |ref| / mag above this: nearly all products of one sign) keeps (a) only
COHERENT = 0.5


def act_fp64(v, act):
    if act == ACT_RELU:
        return v.clamp_min(0)
    if act == ACT_LEAKY01:
        return torch.where(v > 0, v, 0.1 * v)
    return v


def _five(x):
    """[B, H, W, C] or [B, D, H, W, C] -> [B, D, H, W, C] (a view)."""
    return x.unsqueeze(1) if x.dim() == 4 else x


def dense_weight(pc, source=None):
    """float64 [Cout, Cin, kd, kh, kw] of a PackedConv, from fp32 weights the kernels did not produce: its FFMA layout
    [taps * Cin, ldw], or for an operand packed for the tensor cores only (the detector's correlation kernels) the fp32
    rows [Cout, K] it was split from (`source`, K index = tap * Cin + c).  Never from the hi / lo halves the kernels
    read, so a wrong or saturated split shows as a difference."""
    kd, kh, kw = pc.k
    if source is not None:
        v = source.double()[:pc.cout]
        return v.reshape(pc.cout, kd, kh, kw, pc.cin).permute(0, 4, 1, 2, 3).contiguous()
    if pc.w is None:
        raise ValueError('dense_weight: a tensor-core-only operand needs the fp32 rows it was split from')
    w = pc.w.double()[:, :pc.cout].reshape(kd, kh, kw, pc.cin, pc.cout)
    return w.permute(4, 3, 0, 1, 2).contiguous()


def prologue_fp64(x5, prologue, scale, shift, group_rows):
    """x5 float64 [B, D, H, W, Cin] -> the prologue applied to every element (the caller keeps the padding zero)."""
    if prologue == PRO_NONE:
        return x5
    B, D, H, W, C = x5.shape
    if prologue == PRO_CORR:
        return x5 * scale.double().reshape(1, D, H, W, C) + shift.double().reshape(1, 1, 1, 1, C)
    g = torch.arange(B, device=x5.device) // max(int(group_rows), 1)
    v = x5 * scale.double()[g].reshape(B, 1, 1, 1, C) + shift.double()[g].reshape(B, 1, 1, 1, C)
    return v.clamp_min(0) if prologue == PRO_AFFINE_RELU else v


def _as3(t):
    return (t,) * 3 if isinstance(t, int) else tuple(t)


def reference(x, w, bias=None, stride=1, pad=0, prologue=PRO_NONE, scale=None, shift=None, group_rows=1, act=ACT_NONE,
              in_coff=0):
    """x fp32 channels-last [B, (D,) H, W, cs] (channels [in_coff, in_coff + Cin) are read); w [Cout, Cin, kd, kh, kw].
    -> (ref, mag, s), float64 [M, Cout] with M = B * Do * Ho * Wo in the output's row order."""
    cout, cin = w.shape[:2]
    x5 = _five(x)[..., in_coff:in_coff + cin].double()
    xp = prologue_fp64(x5, prologue, scale, shift, group_rows).permute(0, 4, 1, 2, 3)
    w = w.double().to(x.device)
    kw = dict(stride=stride, padding=_as3(pad))
    ref = F.conv3d(xp, w, None, **kw)
    mag = F.conv3d(xp.abs(), w.abs(), None, **kw)
    s = F.conv3d(xp * xp, w * w, None, **kw).sqrt()
    if bias is not None:
        b = bias.double().to(x.device).reshape(1, cout, 1, 1, 1)
        ref, mag = ref + b, mag + b.abs()
    flat = lambda t: t.permute(0, 2, 3, 4, 1).reshape(-1, cout)
    return act_fp64(flat(ref), act), flat(mag), flat(s)


def out_dims(x5_shape, k, stride, pad):
    _, D, H, W, _ = x5_shape
    return tuple((n + 2 * p - kk) // stride + 1 for n, p, kk in zip((D, H, W), _as3(pad), k))


def reference_rows(x, w, rows, bias=None, stride=1, pad=0, prologue=PRO_NONE, scale=None, shift=None, group_rows=1,
                   act=ACT_NONE, in_coff=0, chunk_bytes=1 << 28):
    """reference() at the output rows `rows` (int64 [R]) only: (ref, mag, s) float64 [R, Cout].  The fp64 patches of
    at most chunk_bytes are gathered at a time."""
    cout, cin, kd, kh, kwid = w.shape
    x5 = _five(x)
    B, D, H, W, _ = x5.shape
    Do, Ho, Wo = out_dims(x5.shape, (kd, kh, kwid), stride, pad)
    pd, ph, pw = _as3(pad)
    dev = x.device
    taps = kd * kh * kwid
    wm = w.double().to(dev).permute(2, 3, 4, 1, 0).reshape(taps * cin, cout)         # K = tap * Cin + c
    flat = x5.reshape(-1, x5.shape[-1])
    tz, ty, tx = torch.meshgrid(torch.arange(kd, device=dev), torch.arange(kh, device=dev), torch.arange(kwid, device=dev),
                                indexing='ij')
    tz, ty, tx = tz.reshape(-1), ty.reshape(-1), tx.reshape(-1)
    per = max(1, chunk_bytes // (8 * taps * cin * 3))
    outs = ([], [], [])
    rows = rows.to(dev)
    for r0 in range(0, rows.numel(), per):
        m = rows[r0:r0 + per]
        xo, t = m % Wo, m // Wo
        yo, t = t % Ho, t // Ho
        zo, b = t % Do, t // Do
        zi = zo[:, None] * stride - pd + tz[None]
        yi = yo[:, None] * stride - ph + ty[None]
        xi = xo[:, None] * stride - pw + tx[None]
        inb = (zi >= 0) & (zi < D) & (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
        sp = (zi.clamp(0, D - 1) * H + yi.clamp(0, H - 1)) * W + xi.clamp(0, W - 1)          # [R, taps]
        pix = b[:, None] * (D * H * W) + sp
        p = flat[pix.reshape(-1)][:, in_coff:in_coff + cin].double().reshape(m.numel(), taps, cin)
        if prologue == PRO_CORR:
            p = p * scale.double()[sp.reshape(-1)].reshape(m.numel(), taps, cin) + shift.double().reshape(1, 1, cin)
        elif prologue in (PRO_AFFINE, PRO_AFFINE_RELU):
            g = b // max(int(group_rows), 1)
            p = p * scale.double()[g][:, None] + shift.double()[g][:, None]
            if prologue == PRO_AFFINE_RELU:
                p = p.clamp_min(0)
        p = torch.where(inb[..., None], p, torch.zeros((), dtype=p.dtype, device=dev)).reshape(m.numel(), taps * cin)
        ref, mag, s = p @ wm, p.abs() @ wm.abs(), ((p * p) @ (wm * wm)).sqrt()
        if bias is not None:
            bb = bias.double().to(dev)
            ref, mag = ref + bb, mag + bb.abs()
        for o, v in zip(outs, (act_fp64(ref, act), mag, s)):
            o.append(v)
    return tuple(torch.cat(o) for o in outs)


def coherence(ref, mag):
    """Median over the elements of |ref| / mag: about 1 when all products of a sum share a sign, small for signed data."""
    live = mag > 0
    return float((ref[live].abs() / mag[live]).median()) if bool(live.any()) else 0.0


def measure(y, ref, mag, s):
    """(worst |y - ref| / mag, rms over s > 0 of (y - ref) / s, first element index of the worst (a) ratio)."""
    err = (y.double() - ref).abs()
    ra = err / mag.clamp_min(torch.finfo(torch.float64).tiny)
    ra = torch.where(mag > 0, ra, torch.where(err > 0, torch.full_like(ra, float('inf')), torch.zeros_like(ra)))
    ra = torch.where(torch.isnan(y), torch.full_like(ra, float('inf')), ra)
    live = s > 0
    rb = float(((err[live] / s[live]) ** 2).mean().sqrt()) if bool(live.any()) else 0.0
    worst = int(ra.argmax())
    return float(ra.flatten()[worst]), rb, worst


def check(name, y, ref, mag, s, tau_b=TAU_B_TC, tau_a=TAU_A, class_b=True):
    """Asserts (a) for every element and, with class_b, (b); prints the worst ratios.  y: [M, Cout] (any float dtype).
    Returns (worst (a) ratio / tau_a, (b) rms / tau_b)."""
    a, b, worst = measure(y, ref, mag, s)
    fa, fb = a / tau_a, b / tau_b
    print(f'  {name}: (a) worst |y-ref|/mag {a:.3e} ({fa:.3g} of tau_a)   (b) rms((y-ref)/s) {b:.3e} ({fb:.3g} of tau_b)'
          f'{"" if class_b else " [(b) not asserted]"}')
    if not fa <= 1.0:
        m, n = divmod(worst, y.shape[-1])
        raise AssertionError(f'{name}: (a) |y - ref| <= tau_a * mag fails at row {m}, column {n}: y {float(y[m, n])!r} '
                             f'ref {float(ref[m, n])!r} mag {float(mag[m, n])!r} ({fa:.3g} of the bound)')
    if class_b:
        assert fb <= 1.0, f'{name}: (b) rms((y - ref) / s) = {b:.3e} > tau_b = {tau_b:.1e}'
    return fa, fb


def moments_fp64(y, rows_per_group):
    """Per group of rows_per_group consecutive rows of y [M, C]: float64 [groups, C, 2] of (sum y, sum y^2), and the
    matching error scale (sum |y|, sum y^2)."""
    v = y.double().reshape(-1, rows_per_group, y.shape[-1])
    s1, s2, a1 = v.sum(1), (v * v).sum(1), v.abs().sum(1)
    return torch.stack([s1, s2], -1), torch.stack([a1, s2], -1)


# fp32 moments: per 32-row slice, 8-row fmaf chains combined in shared memory, then fp64 accumulation: about 34 fp32
# roundings on the way to each partial, each bounded by u times the sum of magnitudes
MOMENTS_TOL = 34 * 2.0 ** -24


def check_moments(name, ws, y, rows_per_group):
    """ws float64 [groups, C, 2] (the kernel's) against the fp64 moments of its own y [M, C]: every entry within
    MOMENTS_TOL of its sum of magnitudes.  Returns the worst ratio to that bound."""
    want, scale = moments_fp64(y, rows_per_group)
    assert ws.shape == want.shape, (name, tuple(ws.shape), tuple(want.shape))
    err = (ws.double() - want).abs()
    lim = MOMENTS_TOL * scale + 1e-300
    frac = float((err / lim).max())
    print(f'  {name}: moments worst |ws - fp64(y)| / (34 u sum|.|) = {frac:.3g}')
    assert frac <= 1.0, f'{name}: fused moments off by {frac:.3g} of the fp32 partials bound'
    return frac
