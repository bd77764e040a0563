"""Edges of the 128-row tensor-core tile (two 64-row consumer warpgroups): partial last tiles that end
inside either warpgroup, fused InstanceNorm moments of 32-row groups (four per tile), and split-K from the
one-wave rule, for both operand kinds."""
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
    return x.permute(0, 2, 3, 1).contiguous().cuda()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous().cpu()


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


@pytest.fixture(params=['f16', 'tf32'], autouse=True)
def kind(request):
    old = os.environ.get('G6D_CONV_KIND')
    os.environ['G6D_CONV_KIND'] = request.param
    yield request.param
    if old is None:
        os.environ.pop('G6D_CONV_KIND', None)
    else:
        os.environ['G6D_CONV_KIND'] = old


@pytest.mark.parametrize('rem', [1, 64, 65, 127])
def test_tc_partial_last_tile_persistent(ops, rem):
    """1x1 convolution (persistent kernel), M % 128 = rem: the last tile ends in the first warpgroup's rows,
    at its last row, or in the second warpgroup's."""
    W = 2 * 128 + rem
    x = torch.randn(1, 64, 1, W, generator=g(80)) + 0.5
    w = torch.randn(96, 64, 1, 1, generator=g(81)) * (2 / 64) ** .5
    b = torch.randn(96, generator=g(82))
    ref = F.conv2d(x.double(), w.double(), b.double()).float()
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=0)
    y = ops.conv(nhwc(x), pc)
    assert rel_err(nchw(y), ref) < 5e-6
    assert torch.equal(y, ops.conv(nhwc(x), pc))


# Ho rows of width W = 7 (padded width Wp = 9): the A-reuse kernel enumerates Ho * Wp positions per plane,
# and Ho * 9 % 128 = rem.  The halo (128 + 2 * Wp + 2 = 148 rows) fits its shared-memory budget and the
# valid columns (7 of 9) keep every shape above its 60 % tile-occupancy floor, so all four run on it.
@pytest.mark.parametrize('Ho,rem', [(57, 1), (64, 64), (121, 65), (71, 127)])
def test_tc_partial_last_tile_flat(ops, Ho, rem):
    """3x3 stride-1 convolution (A-reuse kernel): the plane's last tile ends in the first warpgroup's rows,
    at its last row, or in the second warpgroup's."""
    assert Ho * 9 % 128 == rem
    x = torch.randn(2, 64, Ho, 7, generator=g(86)) + 0.5
    w = torch.randn(96, 64, 3, 3, generator=g(87)) * (2 / (9 * 64)) ** .5
    b = torch.randn(96, generator=g(88))
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1).float()
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    y = ops.conv(nhwc(x), pc)
    assert rel_err(nchw(y), ref) < 5e-6
    assert torch.equal(y, ops.conv(nhwc(x), pc))


@pytest.mark.parametrize('B,hw,cin', [(12, 8, 64),       # 6 tiles of 4 groups, no split
                                      (2, 8, 1024)])     # one tile, split-K + the reduce kernel's moments
def test_tc_groups_inside_one_tile(ops, B, hw, cin):
    """Groups of 32 rows (half an 8x8 plane): each 128-row tile adds to four groups' moments."""
    x = torch.randn(B, cin, hw, hw, generator=g(83))
    w = torch.randn(64, cin, 1, 1, generator=g(84)) * cin ** -.5
    b = torch.randn(64, generator=g(85))
    rows = 32
    y, ws = ops.conv(nhwc(x), ops.pack_conv(w.cuda(), b.cuda(), pad=0), stats_rows=rows)
    ref = F.conv2d(x.double(), w.double(), b.double()).float()
    assert rel_err(nchw(y), ref) < 5e-6
    want = ops.instnorm_partial(y, rows_per_group=rows)
    np.testing.assert_allclose(ws.cpu().numpy(), want.cpu().numpy(), rtol=2e-6, atol=1e-4)
