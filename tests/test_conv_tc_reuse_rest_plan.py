"""g6d_conv_tc_plan_ex / g6d_conv_tc_workspace_bytes_ex without a GPU, at the shapes of bench.py's step (10 frames of
480x640, detection scales -1 / -0.5 / 0 / 0.5, 128x128 selector and refiner crops, 64 x 5 selector references, 32
detector references per object) for the layers besides the refiner's that the A-reuse kernel takes without
G6D_TC_REUSE_IM2COL: the detector's row-decomposed correlation, the selector's 16x16 level-0 tower, the crops' and the
detector's VGG maps and the detector heads.  With the flag each of them plans the persistent kernel with the split
input, the A-reuse kernel's BN and K splits, and a workspace of the split-K partials plus 4 bytes per input element;
without it the plan is the A-reuse kernel's, as before."""
import ctypes

import pytest

from gen6d_b200 import _lib

RO = _lib.TC_REUSE_IM2COL


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(B, H, W, Cin, Cout, k=(3, 3), pad=(1, 1), prologue=_lib.PRO_NONE, group_rows=1, max_chain_k=0):
    (kh, kw), (ph, pw) = k, pad
    Ho, Wo = H + 2 * ph - kh + 1, W + 2 * pw - kw + 1
    return _lib.ConvDesc(B=B, D=1, H=H, W=W, Cin=Cin, in_cstride=Cin, in_coff=0, Cout=Cout, kd=1, kh=kh, kw=kw,
                         stride=1, pd=0, ph=ph, pw=pw, Do=1, Ho=Ho, Wo=Wo, out_cstride=Cout, out_coff=0,
                         prologue=prologue, group_rows=group_rows, act=0, max_chain_k=max_chain_k)


def plan(lib, d, flags):
    out = (ctypes.c_int * 4)(-7, -7, -7, -7)
    rc = lib.g6d_conv_tc_plan_ex(ctypes.byref(d), _lib.TC_F16, flags, out)
    return rc, list(out)


def ws(lib, d, flags):
    return lib.g6d_conv_tc_workspace_bytes_ex(ctypes.byref(d), _lib.TC_F16, flags)


RFN = 32                                                   # detector references per object
# the query maps of the four scales (256x320, 352x480, 480x640, 704x928) the correlation kernels of the 120x120
# references slide over: 1/8 with 15 rows, 1/16 with 7 and 1/32 with 3
CORR_MAPS = {15: [(32, 40), (44, 60), (60, 80), (88, 116)], 7: [(16, 20), (22, 30), (30, 40), (44, 58)],
             3: [(8, 10), (11, 15), (15, 20), (22, 29)]}


def corr(k, h, w, n_obj):
    """The row-decomposed k x k correlation of 10 query maps with n_obj objects' references: a 1 x k convolution
    with n_obj * k * RFN output channels, rows padded by k // 2, accumulate chains bounded to 640 K-elements."""
    return desc(10, h, w, 512, n_obj * k * RFN, k=(1, k), pad=(k // 2, k // 2), max_chain_k=640)


CORR = [pytest.param(corr(k, h, w, n), id=f'corr-1x{k}-{h}x{w}-K{n}') for k, hw in CORR_MAPS.items() for h, w in hw
        for n in (1, 2)]
SEL_S = 64 * 5                                             # selector slices (references x in-plane angles)
OTHER = [
    # selector level-0 tower at 16x16: q(.)ref with the first InstanceNorm (per-position scale), then IN+ReLU
    pytest.param(desc(SEL_S, 16, 16, 512, 64, prologue=_lib.PRO_CORR, group_rows=SEL_S), id='sel-tower0-512-64-corr'),
    pytest.param(desc(SEL_S, 16, 16, 64, 64, prologue=_lib.PRO_AFFINE_RELU, group_rows=SEL_S), id='sel-tower0-64-64-inrelu'),
] + [
    # the refiner crops' (70: 10 poses x (query + 6 references)) and the selector crops' VGG at 1/4 and 1/8 of 128^2
    pytest.param(desc(B, s, s, cin, cout), id=f'{who}-vgg-{s}-{cin}-{cout}')
    for who, B in (('ref', 70), ('sel', 10)) for s, cin, cout in ((32, 128, 256), (32, 256, 256), (16, 256, 512),
                                                                  (16, 512, 512))
] + [
    # the detector's 1/16 maps at the three smaller scales and 1/8 at the smallest
    pytest.param(desc(10, h, w, cin, 512), id=f'det-vgg-{h}x{w}-{cin}-512')
    for h, w, cin in ((16, 20, 512), (22, 30, 512), (30, 40, 512), (32, 40, 256), (32, 40, 512))
] + [
    # the detector heads' 3x3 layers at 1/8 of the query
    pytest.param(desc(10, 60, 80, 64, 64), id='det-head-60x80'),
]


@pytest.mark.parametrize('d', CORR + OTHER)
def test_flag_moves_layer_to_split_input_with_same_bn_and_splits(lib, d):
    flags = RO | (_lib.TC_PRENORM if d.prologue else 0)
    rc, ro = plan(lib, d, flags)
    assert rc == 0
    rc, flat = plan(lib, d, flags & ~RO)
    assert rc == 0
    assert flat[0] == 1 and flat[3] == 0                  # without the flag: the A-reuse kernel, as before
    assert ro[0] == 0 and ro[3] == 1                      # with it: persistent, A by TMA im2col from the split copy
    assert ro[1:3] == flat[1:3]                           # the A-reuse kernel's BN and K splits
    assert plan(lib, d, 0)[1] == flat                     # the flag-less call (ops.conv's default) is unchanged
    M = d.B * d.Ho * d.Wo
    partials = ro[2] * M * d.Cout * 4 if ro[2] > 1 else 0
    assert ws(lib, d, flags & ~RO) == partials
    assert ws(lib, d, flags) == (partials + 255) // 256 * 256 + 4 * d.B * d.H * d.W * d.Cin


@pytest.mark.parametrize('n_obj', [1, 2])
def test_largest_correlation_keeps_eight_chain_bounded_splits(lib, n_obj):
    """K = 15 * 512 = 7680 with chains of 640: eight splits, one channel block (15 K-blocks) each."""
    d = corr(15, 88, 116, n_obj)
    assert plan(lib, d, RO)[1] == [0, 128, 8, 1]
    assert plan(lib, d, 0)[1] == [1, 128, 8, 0]


def test_selector_tower_keeps_one_split_for_the_moments(lib):
    """No K split: the fused moments come from flat_moments_kernel over the A-reuse kernel's slices."""
    d = desc(SEL_S, 16, 16, 512, 64, prologue=_lib.PRO_CORR, group_rows=SEL_S)
    assert plan(lib, d, RO | _lib.TC_PRENORM)[1] == [0, 64, 1, 1]
    assert lib.g6d_conv_tc_stats_supported(ctypes.byref(d), _lib.TC_F16, SEL_S * 256) == 1
