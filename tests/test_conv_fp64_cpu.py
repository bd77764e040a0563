"""The fp64 convolution reference of conv_fp64_ref.py against a direct per-element loop in numpy, without a GPU: the
prologues (affine per norm group, affine + ReLU, the selector's per-position correlation scale) on in-bounds elements
only, input channel slices, stride and padding in 2-D and 3-D, bias and activations, and the error scales mag and s.
Both forms are checked (whole-tensor convolution and gathered rows), and the weight layouts the reference reads back
from a PackedConv."""
import types

import numpy as np
import pytest
import torch

import conv_fp64_ref as R


def loop_reference(x5, w, bias, stride, pad, prologue, scale, shift, group_rows, act, in_coff):
    """x5 [B, D, H, W, cs] numpy -> (ref, mag, s) [B, Do, Ho, Wo, Cout] by one explicit sum per output element."""
    B, D, H, W, _ = x5.shape
    cout, cin, kd, kh, kw = w.shape
    pd, ph, pw = pad
    Do, Ho, Wo = ((D + 2 * pd - kd) // stride + 1, (H + 2 * ph - kh) // stride + 1, (W + 2 * pw - kw) // stride + 1)
    ref, mag, s2 = (np.zeros((B, Do, Ho, Wo, cout)) for _ in range(3))
    for b in range(B):
        for zo in range(Do):
            for yo in range(Ho):
                for xo in range(Wo):
                    for o in range(cout):
                        acc = am = sq = 0.0
                        for kz in range(kd):
                            for ky in range(kh):
                                for kx in range(kw):
                                    zi, yi, xi = zo * stride - pd + kz, yo * stride - ph + ky, xo * stride - pw + kx
                                    if not (0 <= zi < D and 0 <= yi < H and 0 <= xi < W):
                                        continue
                                    for c in range(cin):
                                        v = float(x5[b, zi, yi, xi, in_coff + c])
                                        if prologue == R.PRO_CORR:
                                            v = v * scale[(zi * H + yi) * W + xi, c] + shift[c]
                                        elif prologue in (R.PRO_AFFINE, R.PRO_AFFINE_RELU):
                                            g = b // group_rows
                                            v = v * scale[g, c] + shift[g, c]
                                            if prologue == R.PRO_AFFINE_RELU:
                                                v = max(v, 0.0)
                                        p = v * float(w[o, c, kz, ky, kx])
                                        acc += p; am += abs(p); sq += p * p
                        if bias is not None:
                            acc += float(bias[o]); am += abs(float(bias[o]))
                        if act == R.ACT_RELU:
                            acc = max(acc, 0.0)
                        elif act == R.ACT_LEAKY01:
                            acc = acc if acc > 0 else 0.1 * acc
                        ref[b, zo, yo, xo, o], mag[b, zo, yo, xo, o], s2[b, zo, yo, xo, o] = acc, am, sq
    return ref, mag, np.sqrt(s2)


CASES = [
    # (x shape [B, (D,) H, W, cs], Cin, Cout, k, stride, pad, prologue, group_rows, act, in_coff, bias)
    pytest.param((2, 5, 6, 8), 8, 3, (1, 3, 3), 1, (0, 1, 1), R.PRO_NONE, 1, R.ACT_NONE, 0, True, id='2d-3x3'),
    pytest.param((3, 7, 5, 12), 4, 2, (1, 3, 3), 2, (0, 1, 1), R.PRO_AFFINE, 2, R.ACT_RELU, 4, True, id='2d-s2-affine-slice'),
    pytest.param((4, 4, 5, 8), 8, 3, (1, 3, 3), 1, (0, 0, 0), R.PRO_AFFINE_RELU, 1, R.ACT_LEAKY01, 0, False, id='2d-valid-affrelu'),
    pytest.param((3, 4, 4, 8), 8, 2, (1, 3, 3), 1, (0, 1, 1), R.PRO_CORR, 3, R.ACT_NONE, 0, True, id='2d-corr'),
    pytest.param((2, 3, 4, 5, 4), 4, 2, (3, 3, 3), 2, (1, 1, 1), R.PRO_AFFINE, 1, R.ACT_RELU, 0, True, id='3d-s2-affine'),
    pytest.param((1, 1, 4, 5, 8), 4, 3, (3, 3, 3), 1, (1, 1, 1), R.PRO_CORR, 1, R.ACT_NONE, 4, False, id='3d-d1-kd3-corr-slice'),
    pytest.param((2, 3, 3, 4), 4, 2, (1, 1, 1), 1, (0, 0, 0), R.PRO_NONE, 1, R.ACT_LEAKY01, 0, True, id='1x1'),
    pytest.param((1, 3, 9, 4), 4, 2, (1, 1, 5), 1, (0, 0, 2), R.PRO_NONE, 1, R.ACT_NONE, 0, False, id='1x5-row'),
]


@pytest.mark.parametrize('shape, cin, cout, k, stride, pad, prologue, group_rows, act, in_coff, bias', CASES)
def test_reference_matches_loop(shape, cin, cout, k, stride, pad, prologue, group_rows, act, in_coff, bias):
    gen = torch.Generator().manual_seed(sum(shape) + cin * 7 + prologue)
    x = torch.randn(*shape, generator=gen)
    x5 = x.unsqueeze(1) if x.dim() == 4 else x
    B, D, H, W = x5.shape[:4]
    w = torch.randn(cout, cin, *k, generator=gen)
    b = torch.randn(cout, generator=gen) if bias else None
    scale = shift = None
    if prologue == R.PRO_CORR:
        scale, shift = torch.rand(D * H * W, cin, generator=gen) + 0.5, torch.randn(cin, generator=gen)
    elif prologue != R.PRO_NONE:
        groups = (B + group_rows - 1) // group_rows
        scale, shift = torch.rand(groups, cin, generator=gen) + 0.5, torch.randn(groups, cin, generator=gen)
    kw = dict(stride=stride, pad=pad, prologue=prologue, scale=scale, shift=shift, group_rows=group_rows, act=act,
              in_coff=in_coff)
    want = loop_reference(x5.numpy(), w.numpy(), None if b is None else b.numpy(), stride, pad, prologue,
                          None if scale is None else scale.double().numpy(), None if shift is None else shift.double().numpy(),
                          group_rows, act, in_coff)
    got = R.reference(x, w, b, **kw)
    M = want[0].size // cout
    for name, g, e in zip(('ref', 'mag', 's'), got, want):
        assert tuple(g.shape) == (M, cout), name
        np.testing.assert_allclose(g.numpy(), e.reshape(M, cout), rtol=1e-12, atol=1e-12, err_msg=name)
    rows = torch.tensor(sorted({0, M - 1, M // 2, M // 3}))
    got_rows = R.reference_rows(x, w, rows, b, chunk_bytes=8 * cin * 3 * k[0] * k[1] * k[2] * 2, **kw)   # 2 rows per chunk
    for name, g, e in zip(('ref', 'mag', 's'), got_rows, want):
        np.testing.assert_allclose(g.numpy(), e.reshape(M, cout)[rows.numpy()], rtol=1e-12, atol=1e-12, err_msg=name)
    assert bool((got[1] >= got[0].abs() - 1e-12).all() if act == R.ACT_NONE else True)


def test_padding_stays_zero_under_the_prologue():
    """A shift that would make padded taps non-zero must not reach them: with x = 0 and shift = 1 the border outputs
    see fewer in-bounds taps than the interior ones."""
    x = torch.zeros(1, 4, 4, 4)
    w = torch.ones(1, 4, 1, 3, 3)
    ref, _, _ = R.reference(x, w, pad=(0, 1, 1), prologue=R.PRO_AFFINE, scale=torch.ones(1, 4), shift=torch.ones(1, 4))
    grid = ref.reshape(4, 4)
    assert float(grid[0, 0]) == 4 * 4 and float(grid[1, 1]) == 9 * 4 and float(grid[0, 1]) == 6 * 4


def test_measure_flags_a_single_small_element():
    """(a) is per element: one wrong value at an element with a small magnitude fails even when the normwise error is
    tiny, and NaN always fails."""
    ref = torch.tensor([[1000.0, 1e-3]], dtype=torch.float64)
    mag = ref.abs() * 2
    s = ref.abs()
    y = ref.clone()
    y[0, 1] += 1e-6
    a, _, worst = R.measure(y, ref, mag, s)
    assert worst == 1 and a > R.TAU_A
    assert float((y - ref).abs().max() / ref.abs().max()) < 1e-9
    y[0, 1] = float('nan')
    assert R.measure(y, ref, mag, s)[0] == float('inf')
    with pytest.raises(AssertionError):
        R.check('nan', y, ref, mag, s)


@pytest.mark.parametrize('kind', [R.TC_TF32, R.TC_F16])
def test_dense_weight_from_packed_layouts(kind):
    """dense_weight reads the FFMA layout [taps * Cin, ldw] and, for a tensor-core-only operand of either kind, the fp32
    rows [Cout, K] it was split from (K = tap * Cin + c), never its hi / lo halves; both give the original weight, and
    without either it refuses."""
    gen = torch.Generator().manual_seed(3 + kind)
    cout, cin, k = 18, 64, (1, 3, 2)
    w = torch.randn(cout, cin, *k, generator=gen)
    wk = w.permute(2, 3, 4, 1, 0).reshape(6 * cin, cout)          # K = tap * Cin + c
    packed = torch.zeros(6 * cin, (cout + 3) // 4 * 4)
    packed[:, :cout] = wk
    pc = types.SimpleNamespace(w=packed, k=k, cin=cin, cout=cout, kind=kind, w_hi=None, w_lo=None)
    assert torch.equal(R.dense_weight(pc), w.double())
    pc.w = None
    assert torch.equal(R.dense_weight(pc, source=wk.T.contiguous()), w.double())
    with pytest.raises(ValueError):
        R.dense_weight(pc)
