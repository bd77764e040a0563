"""G6D_TC_FOLD_SPLITS in the planner, without a GPU, at the shapes of bench.py's step (10 frames of 480x640, detection
scales -1 / -0.5 / 0 / 0.5, 128x128 crops, 32 detector references per object): which layers fold, that the K splits
stay what they were, that a folded plan's workspace is the split input alone, and that the flag changes nothing where
folding does not apply (producer-warp path, tf32, one split, grids whose splits fill a wave tail)."""
import ctypes

import pytest

from gen6d_b200 import _lib
from test_conv_tc_reuse_rest_plan import CORR_MAPS, corr, desc

RO, FOLD = _lib.TC_REUSE_IM2COL, _lib.TC_FOLD_SPLITS


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def plan(lib, d, flags, kind=_lib.TC_F16):
    out = (ctypes.c_int * 5)(-7, -7, -7, -7, -7)
    rc = lib.g6d_conv_tc_plan_v2(ctypes.byref(d), kind, flags, out, 5)
    return rc, list(out)


def ws(lib, d, flags, kind=_lib.TC_F16):
    return lib.g6d_conv_tc_workspace_bytes_ex(ctypes.byref(d), kind, flags)


def vol(S, cin, cout, pro=_lib.PRO_NONE, B=10):
    return _lib.ConvDesc(B=B, D=S, H=S, W=S, Cin=cin, in_cstride=cin, in_coff=0, Cout=cout, kd=3, kh=3, kw=3, stride=1,
                         pd=1, ph=1, pw=1, Do=S, Ho=S, Wo=S, out_cstride=cout, out_coff=0, prologue=pro, group_rows=1, act=0,
                         max_chain_k=0)


# the detector's VGG at 1/4, 1/8 and 1/16 of the four scales (256x320, 352x480, 480x640, 704x928)
DET_VGG = ([(f'det-vgg4-{h}x{w}-{ci}', desc(10, h, w, ci, 256)) for h, w in ((64, 80), (88, 120), (120, 160), (176, 232))
            for ci in (128, 256)]
           + [(f'det-vgg8-{h}x{w}-{ci}', desc(10, h, w, ci, 512)) for h, w in CORR_MAPS[15] for ci in (256, 512)]
           + [(f'det-vgg16-{h}x{w}', desc(10, h, w, 512, 512)) for h, w in CORR_MAPS[7]])
CORR = [(f'corr-1x{k}-{h}x{w}-K{n}', corr(k, h, w, n)) for k, hw in CORR_MAPS.items() for h, w in hw for n in (1, 2)]
CROPS = [(f'{who}-vgg-{s}-{ci}-{co}', desc(B, s, s, ci, co)) for who, B in (('ref', 70), ('sel', 10))
         for s, ci, co in ((32, 128, 256), (32, 256, 256), (16, 256, 512), (16, 512, 512))]
# the refiner's volume net: the 32^3 embeddings (64 + 64 channels in, then IN+ReLU), the 16^3 / 8^3 / 4^3 trunk
REFINER = [('ref-vol32-128-64', vol(32, 128, 64)), ('ref-vol32-64-64', vol(32, 64, 64, _lib.PRO_AFFINE_RELU)),
           ('ref-vol16-64-128', vol(16, 64, 128)), ('ref-vol16-128-128', vol(16, 128, 128, _lib.PRO_AFFINE_RELU)),
           ('ref-vol8-128-256', vol(8, 128, 256, _lib.PRO_AFFINE_RELU)), ('ref-vol8-256-256', vol(8, 256, 256, _lib.PRO_AFFINE_RELU)),
           ('ref-vol4-256-512', vol(4, 256, 512, _lib.PRO_AFFINE_RELU)), ('ref-vol4-512-512', vol(4, 512, 512, _lib.PRO_AFFINE_RELU))]
SEL_TOWER = [('sel-tower0-512-64', desc(320, 16, 16, 512, 64, prologue=_lib.PRO_CORR, group_rows=320))]

FOLDED = {
    'corr-1x15-32x40-K1', 'corr-1x15-32x40-K2', 'corr-1x15-44x60-K1', 'corr-1x15-44x60-K2', 'corr-1x15-60x80-K1',
    'corr-1x15-60x80-K2', 'corr-1x15-88x116-K1', 'corr-1x15-88x116-K2', 'corr-1x7-22x30-K1', 'corr-1x7-22x30-K2',
    'corr-1x7-30x40-K1', 'corr-1x7-30x40-K2', 'corr-1x7-44x58-K1', 'corr-1x7-44x58-K2', 'corr-1x3-22x29-K2',
    'det-vgg4-64x80-256', 'det-vgg4-88x120-256', 'det-vgg4-120x160-256', 'det-vgg4-176x232-256',
    'det-vgg8-32x40-256', 'det-vgg8-44x60-256', 'det-vgg8-44x60-512', 'det-vgg8-60x80-256', 'det-vgg8-60x80-512',
    'det-vgg8-88x116-256', 'det-vgg8-88x116-512', 'det-vgg16-16x20', 'det-vgg16-30x40', 'det-vgg16-44x58',
    'ref-vgg-32-256-256', 'ref-vgg-16-256-512', 'sel-vgg-16-256-512', 'ref-vol8-128-256',
}
ALL = CORR + DET_VGG + CROPS + REFINER + SEL_TOWER


@pytest.mark.parametrize('name, d', [pytest.param(n, d, id=n) for n, d in ALL])
def test_fold_decision_at_bench_shapes(lib, name, d):
    base = RO | (_lib.TC_PRENORM if d.prologue else 0)
    rc, p = plan(lib, d, base)
    assert rc == 0 and p[4] == 0
    rc, f = plan(lib, d, base | FOLD)
    assert rc == 0
    assert f[:4] == p[:4]                                 # same kernel, BN, K splits and A operand
    assert f[4] == (1 if name in FOLDED else 0)
    if f[4]:
        assert p[0] == 0 and p[3] == 1 and p[2] > 1       # persistent kernel, split input, K splits
        M = d.B * d.Do * d.Ho * d.Wo
        T, S = -(-M // 128) * -(-d.Cout // p[1]), p[2]
        assert -(-T // 132) * S <= 1.15 * -(-T * S // 132)           # S-chain tiles add at most 15 % of waves
        assert ws(lib, d, base | FOLD) == 4 * d.B * d.D * d.H * d.W * d.Cin       # the split input alone
        assert ws(lib, d, base) == (p[2] * M * d.Cout * 4 + 255) // 256 * 256 + 4 * d.B * d.D * d.H * d.W * d.Cin
    else:
        assert ws(lib, d, base | FOLD) == ws(lib, d, base)


def test_largest_correlation_folds_its_eight_splits(lib):
    """K = 15 * 512 = 7680 in chains of 640: 8 splits, 3700 tiles of 128 x 128; the 1.9 GB of partials go."""
    d = corr(15, 88, 116, 1)
    assert plan(lib, d, RO | FOLD)[1] == [0, 128, 8, 1, 1]
    assert ws(lib, d, RO) - ws(lib, d, RO | FOLD) == 8 * 10 * 102 * 116 * 480 * 4


def test_no_effect_without_split_input_or_splits(lib):
    # producer-warp path (stride 2; a prologue without G6D_TC_PRENORM), tf32, one split, a grid whose splits fill a wave tail
    s2 = _lib.ConvDesc(B=10, D=1, H=176, W=232, Cin=256, in_cstride=256, in_coff=0, Cout=256, kd=1, kh=3, kw=3, stride=2,
                       pd=0, ph=1, pw=1, Do=1, Ho=88, Wo=116, out_cstride=256, out_coff=0, prologue=0, group_rows=1, act=0,
                       max_chain_k=0)
    pro = desc(10, 88, 116, 512, 512, prologue=_lib.PRO_AFFINE_RELU, group_rows=10)
    one = desc(10, 120, 160, 128, 256)
    tail = desc(10, 22, 30, 512, 512)                     # 208 tiles, 3 splits: 6 waves folded against 5
    for d, kind in ((s2, _lib.TC_F16), (pro, _lib.TC_F16), (desc(10, 88, 116, 512, 512), _lib.TC_TF32), (one, _lib.TC_F16),
                    (tail, _lib.TC_F16)):
        for flags in (0, RO):
            rc, p = plan(lib, d, flags, kind)
            rc2, f = plan(lib, d, flags | FOLD, kind)
            assert rc == rc2 == 0
            assert f == p and f[4] == 0
            assert ws(lib, d, flags | FOLD, kind) == ws(lib, d, flags, kind)
            buf = (ctypes.c_int * 4)()
            assert lib.g6d_conv_tc_plan_ex(ctypes.byref(d), kind, flags | FOLD, buf) == 0 and list(buf) == p[:4]
    assert plan(lib, s2, FOLD)[1][2] > 1 and plan(lib, pro, FOLD)[1][2] > 1 and plan(lib, tail, RO | FOLD)[1][2] > 1


def test_other_bits_are_still_rejected(lib):
    d = corr(15, 88, 116, 1)
    for bad in (2, 8, 16, 64):
        assert plan(lib, d, RO | FOLD | bad)[0] != 0


def test_plan_v2_writes_at_most_n_values(lib):
    d = corr(15, 88, 116, 1)
    out = (ctypes.c_int * 5)(-7, -7, -7, -7, -7)
    assert lib.g6d_conv_tc_plan_v2(ctypes.byref(d), _lib.TC_F16, RO | FOLD, out, 3) == 0
    assert list(out) == [0, 128, 8, -7, -7]
