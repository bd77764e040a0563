"""The wgmma split-operand convolution (g6d_conv_tc) against torch fp64 CPU and against the FFMA
path, for both operand kinds (G6D_TC_F16: fp16 hi + 2^11-scaled fp16 lo, the default; G6D_TC_TF32: tf32
hi/lo): it must be fp32-faithful (error ~1e-6 relative; a single TF32 or fp16 product would be ~5e-4)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def g(seed):
    gen = torch.Generator(device='cpu')
    gen.manual_seed(seed)
    return gen


def nhwc(x):
    nd = x.dim()
    return x.permute(0, *range(2, nd), 1).contiguous().cuda()


def nchw(x):
    nd = x.dim()
    return x.permute(0, nd - 1, *range(1, nd - 1)).contiguous().cpu()


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


@pytest.fixture(params=['f16', 'tf32'], autouse=True)
def kind(request):
    """Every test runs once per operand kind (read by ops.pack_conv / ops.split_operand at pack time)."""
    old = os.environ.get('G6D_CONV_KIND')
    os.environ['G6D_CONV_KIND'] = request.param
    yield request.param
    if old is None:
        os.environ.pop('G6D_CONV_KIND', None)
    else:
        os.environ['G6D_CONV_KIND'] = old


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize('B,H,W,cin,cout', [(1, 16, 16, 32, 32), (2, 17, 23, 64, 64), (1, 32, 40, 128, 256),
                                            (3, 8, 8, 512, 48), (1, 60, 80, 64, 128), (5, 4, 4, 256, 256)])
def test_tc_conv2d_matches_fp32(ops, kind, B, H, W, cin, cout):
    x = torch.randn(B, cin, H, W, generator=g(1)) + 0.5
    w = torch.randn(cout, cin, 3, 3, generator=g(2)) * (2 / (9 * cin)) ** .5
    b = torch.randn(cout, generator=g(3))
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1)).float()
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    assert pc.w_hi is not None
    assert pc.kind == (1 if (kind == 'f16' and cin % 64 == 0) else 0)
    os.environ['G6D_CONV_PATH'] = 'tc'
    y_tc = nchw(ops.conv(nhwc(x), pc, act=ops.ACT_RELU))
    os.environ['G6D_CONV_PATH'] = 'ffma'
    y_ff = nchw(ops.conv(nhwc(x), pc, act=ops.ACT_RELU))
    os.environ['G6D_CONV_PATH'] = 'tc'
    e_tc, e_ff = rel_err(y_tc, ref), rel_err(y_ff, ref)
    print(f'rel err vs fp64: tc {e_tc:.2e} ffma {e_ff:.2e}')
    assert e_tc < 5e-6, e_tc          # fp32-faithful (plain TF32 would be ~5e-4)
    assert e_ff < 5e-6


@pytest.mark.parametrize('stride', [1, 2])
def test_tc_conv3d(ops, stride):
    x = torch.randn(2, 64, 8, 8, 8, generator=g(4))
    w = torch.randn(128, 64, 3, 3, 3, generator=g(5)) * (2 / (27 * 64)) ** .5
    b = torch.randn(128, generator=g(6))
    ref = F.conv3d(x.double(), w.double(), b.double(), stride=stride, padding=1).float()
    y = nchw(ops.conv(nhwc(x), ops.pack_conv(w.cuda(), b.cuda(), stride=stride, pad=1)))
    assert rel_err(y, ref) < 5e-6


def test_tc_splitk_correlation(ops):
    q = torch.randn(1, 512, 12, 16, generator=g(7)).abs()
    r = torch.randn(32, 512, 15, 15, generator=g(8)).abs()
    ref = F.conv2d(q.double(), r.double(), padding=7).float()
    rk = r.permute(0, 2, 3, 1).contiguous().cuda()
    flat = rk.reshape(32, -1)
    pc = ops.PackedConv(ops.transpose_to_packed(flat), None, 512, 32, (1, 15, 15), 1, (0, 7, 7), max_chain_k=640)
    pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, ops.tc_kind_for(512))
    y = nchw(ops.conv(nhwc(q), pc))
    assert rel_err(y, ref) < 5e-6


@pytest.mark.parametrize('k,rfn,H,W', [(15, 32, 12, 16), (7, 32, 9, 11), (3, 64, 6, 5)])
def test_tc_row_decomposed_correlation(ops, k, rfn, H, W):
    """The detector's sliding inner product as a 1 x k convolution with k*rfn output channels + the row sum
    (g6d_det_corr_rowsum) equals F.conv2d with the k x k kernels (detector.py:222-224)."""
    q = torch.randn(2, 512, H, W, generator=g(40)).abs()
    r = torch.randn(rfn, 512, k, k, generator=g(41)).abs()
    ref = F.conv2d(q.double(), r.double(), padding=k // 2).float()
    f = r.permute(0, 2, 3, 1).contiguous().cuda()                       # [rfn, ky, kx, c] as the detector caches them
    flat = f.permute(1, 0, 2, 3).reshape(k * rfn, k * 512).contiguous()
    pc = ops.PackedConv(None, None, 512, k * rfn, (1, 1, k), 1, (0, k // 2, k // 2), max_chain_k=640)
    pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, ops.tc_kind_for(512))
    part = ops.conv(nhwc(q), pc)
    assert tuple(part.shape) == (2, H + k - 1, W, k * rfn)
    y = nchw(ops.det_corr_rowsum(part, k, rfn))
    assert rel_err(y, ref) < 5e-6


@pytest.mark.parametrize('relu', [False, True])
def test_tc_affine_prologue(ops, relu):
    x = torch.randn(3, 64, 10, 12, generator=g(12)) * 2 + 1
    w = torch.randn(32, 64, 3, 3, generator=g(13)) * 0.05
    xn = F.instance_norm(x.double())
    xn = F.relu(xn) if relu else xn
    ref = F.conv2d(xn, w.double(), None, padding=1).float()
    xc = nhwc(x)
    ps, pb = ops.instnorm_stats(xc, rows_per_group=10 * 12)
    y = ops.conv(xc, ops.pack_conv(w.cuda(), None, pad=1), prologue=ops.PRO_AFFINE_RELU if relu else ops.PRO_AFFINE,
                 pro_scale=ps, pro_shift=pb, group_rows=1)
    assert rel_err(nchw(y), ref) < 2e-5


def test_tc_corr_prologue_and_channel_offsets(ops):
    """Selector first-tower conv: x*scale[pos,c] + shift[c] on in-bounds taps; output into a concat buffer."""
    S, h, w_, cin, cout = 6, 8, 8, 512, 64
    x = torch.rand(S, cin, h, w_, generator=g(20))
    scale = torch.rand(h * w_, cin, generator=g(21)) + 0.5
    shift = torch.randn(cin, generator=g(22)) * 0.1
    wt = torch.randn(cout, cin, 1, 3, 3, generator=g(23)) * 0.02
    b = torch.randn(cout, generator=g(24))
    xs = x.double() * scale.T.reshape(1, cin, h, w_).double() + shift.reshape(1, cin, 1, 1).double()
    ref = F.conv2d(xs, wt[:, :, 0].double(), b.double(), padding=1).float()
    out = torch.zeros(S, h, w_, 192, device='cuda')
    ops.conv(nhwc(x), ops.pack_conv(wt.cuda(), b.cuda(), pad=(0, 1, 1)), prologue=ops.PRO_CORR, pro_scale=scale.cuda(),
             pro_shift=shift.cuda(), group_rows=S, out=out, out_coff=64)
    assert rel_err(nchw(out[..., 64:128].contiguous()), ref) < 5e-6
    assert float(out[..., :64].abs().max()) == 0 and float(out[..., 128:].abs().max()) == 0


@pytest.mark.parametrize('gain', [1e-3, 1.0, 3e2])
def test_tc_dynamic_range(ops, kind, gain):
    """Activations x gain, weights / gain: the fp16 kind keeps fp32-level accuracy over the range the
    network's tensor-core operands live in (BN-folded weights, post-ReLU / normalised activations)."""
    x = (torch.randn(1, 128, 24, 24, generator=g(30)).abs() * gain)
    w = torch.randn(64, 128, 3, 3, generator=g(31)) * (2 / (9 * 128)) ** .5 / gain
    ref = F.conv2d(x.double(), w.double(), None, padding=1).float()
    y = nchw(ops.conv(nhwc(x), ops.pack_conv(w.cuda(), None, pad=1)))
    e = rel_err(y, ref)
    print(f'{kind} gain {gain:g}: rel err vs fp64 {e:.2e}')
    assert e < 5e-6


def test_tc_f16_saturates_instead_of_overflowing(ops, kind):
    """Beyond the fp16 range the conversion saturates (finite result, large error) -- never inf / NaN."""
    x = torch.full((1, 64, 8, 8), 1e6)
    w = torch.full((32, 64, 1, 1), 1e-3)
    y = ops.conv(nhwc(x), ops.pack_conv(w.cuda(), None, pad=0))
    assert torch.isfinite(y).all()
    if kind == 'tf32':
        assert rel_err(nchw(y), torch.full((1, 32, 8, 8), 64e3)) < 1e-5


@pytest.mark.parametrize('case', ['flat2d', 'strided3d', 'splitk', 'onexone'])
def test_tc_fused_output_statistics(ops, case):
    """The InstanceNorm moments a convolution's epilogue (or its split-K reduce) accumulates equal the
    separate pass over its output (g6d_instnorm_partial), and the resulting scale / shift match torch."""
    if case == 'flat2d':
        x = torch.randn(3, 64, 16, 16, generator=g(50)); w = torch.randn(64, 64, 3, 3, generator=g(51)) * 0.05; stride, rows = 1, 256
    elif case == 'strided3d':
        x = torch.randn(2, 64, 8, 8, 8, generator=g(52)); w = torch.randn(128, 64, 3, 3, 3, generator=g(53)) * 0.03; stride, rows = 2, 64
    elif case == 'splitk':
        x = torch.randn(2, 512, 4, 4, 4, generator=g(54)); w = torch.randn(512, 512, 3, 3, 3, generator=g(55)) * 0.01; stride, rows = 1, 64
    else:
        x = torch.randn(20, 768, 4, 4, generator=g(56)); w = torch.randn(512, 768, 1, 1, generator=g(57)) * 0.03; stride, rows = 1, 320
    b = torch.randn(w.shape[0], generator=g(58))
    pc = ops.pack_conv(w.cuda(), b.cuda(), stride=stride, pad=1 if w.shape[-1] == 3 else 0)
    y, ws = ops.conv(nhwc(x), pc, stats_rows=rows)
    want = ops.instnorm_partial(y, rows_per_group=rows)
    assert ws.shape == want.shape
    np.testing.assert_allclose(ws.cpu().numpy(), want.cpu().numpy(), rtol=2e-6, atol=1e-4)
    ps, pb = ops.instnorm_finalize(ws, rows, 1e-5)
    conv = F.conv3d if x.dim() == 5 else F.conv2d
    ref = conv(x.double(), w.double(), b.double(), stride=stride, padding=1 if w.shape[-1] == 3 else 0)
    flat = ref.flatten(2).transpose(1, 2).reshape(-1, rows, w.shape[0])          # [groups, rows, C] (groups of whole samples)
    mean, var = flat.mean(1), flat.var(1, unbiased=False)
    np.testing.assert_allclose(ps.cpu().numpy(), (1 / torch.sqrt(var + 1e-5)).float().numpy(), rtol=2e-5)
    np.testing.assert_allclose(pb.cpu().numpy(), (-mean / torch.sqrt(var + 1e-5)).float().numpy(), rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize('B,hw,cin,cout', [(320, 8, 128, 128),    # 160 tiles on the persistent grid
                                           (320, 4, 256, 256),    # 80 tiles
                                           (150, 8, 128, 192),    # 75 x 2 tiles, the second N tile half empty
                                           (80, 4, 256, 256),     # 20 tiles -> uniform split-K
                                           (1, 8, 512, 512)])     # one M tile, four N tiles (uniform split-K)
def test_tc_tile_counts_that_do_not_divide_the_grid(ops, B, hw, cin, cout):
    """Persistent kernel with tile counts that do not divide over its persistent CTAs (a partial last round, or a short
    grid with uniform split-K + the reduce kernel), InstanceNorm prologue and fused output moments: fp32-faithful
    and bit-reproducible."""
    x = torch.randn(B, cin, hw, hw, generator=g(70)) * 2 + 1
    w = torch.randn(cout, cin, 3, 3, generator=g(71)) * (2 / (9 * cin)) ** .5
    b = torch.randn(cout, generator=g(72))
    xn = F.relu(F.instance_norm(x.double()))
    ref = F.conv2d(xn, w.double(), b.double(), padding=1).float()
    xc = nhwc(x)
    ps, pb = ops.instnorm_stats(xc, rows_per_group=hw * hw)
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    rows = hw * hw if (hw * hw) % 32 == 0 else 32
    kw = dict(prologue=ops.PRO_AFFINE_RELU, pro_scale=ps, pro_shift=pb, group_rows=1)
    if (B * hw * hw) % rows == 0:
        y, ws = ops.conv(xc, pc, stats_rows=rows, **kw)
        want = ops.instnorm_partial(y, rows_per_group=rows)
        np.testing.assert_allclose(ws.cpu().numpy(), want.cpu().numpy(), rtol=2e-6, atol=1e-4)
    else:
        y = ops.conv(xc, pc, **kw)
    assert rel_err(nchw(y), ref) < 2e-5
    y2 = ops.conv(xc, pc, **kw)
    assert torch.equal(y, y2)
