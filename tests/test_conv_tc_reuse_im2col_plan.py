"""g6d_conv_tc_plan_ex / g6d_conv_tc_workspace_bytes_ex without a GPU: G6D_TC_REUSE_IM2COL moves the layers the
A-reuse kernel would take onto the persistent kernel with the split input, keeping that kernel's BN and K splits; it
gives 3-D layers on the persistent kernel the split input through a rank-5 im2col map; and it changes nothing where
the split input cannot apply (1x1, stride 2, tf32, a prologue without G6D_TC_PRENORM, box corners out of the
rank-5 range).  Bad flags and descriptors are rejected with the existing messages."""
import ctypes

import pytest

from gen6d_b200 import _lib

G6D_EINVAL = -1
RO = _lib.TC_REUSE_IM2COL
BOTH = _lib.TC_PRENORM | _lib.TC_REUSE_IM2COL


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(S=32, Cin=64, Cout=64, B=2, D=None, k=3, pad=1, stride=1, prologue=_lib.PRO_NONE):
    """A cubic S^3 volume (D = S) or, with D=1, a 2-D S x S plane; k^3 (k^2) filter, group_rows 1."""
    D = S if D is None else D
    kd, pd = (k, pad) if D > 1 else (1, 0)
    o = (S + 2 * pad - k) // stride + 1
    od = (D + 2 * pd - kd) // stride + 1
    return _lib.ConvDesc(B=B, D=D, H=S, W=S, Cin=Cin, in_cstride=Cin, in_coff=0, Cout=Cout, kd=kd, kh=k, kw=k,
                         stride=stride, pd=pd, ph=pad, pw=pad, Do=od, Ho=o, Wo=o, out_cstride=Cout, out_coff=0,
                         prologue=prologue, group_rows=1, act=0, max_chain_k=0)


def plan(lib, d, kind, flags):
    out = (ctypes.c_int * 4)(-7, -7, -7, -7)
    rc = lib.g6d_conv_tc_plan_ex(ctypes.byref(d), kind, flags, out)
    return rc, list(out)


def ws(lib, d, kind, flags):
    return lib.g6d_conv_tc_workspace_bytes_ex(ctypes.byref(d), kind, flags)


def split_bytes(d):
    return d.B * d.D * d.H * d.W * d.Cin * 4


# the refiner's layers the A-reuse kernel takes: the 32^3 embeds and trunk conv0, trunk conv2 at 16^3, the feature
# branches at 32^2 and 16^2 (70 crops)
REUSE = [dict(S=32, Cin=256), dict(S=32, Cin=128), dict(S=32, Cin=64, prologue=_lib.PRO_AFFINE_RELU),
         dict(S=16, Cin=128, Cout=128, prologue=_lib.PRO_AFFINE_RELU),
         dict(S=32, D=1, B=70, Cin=256), dict(S=32, D=1, B=70, Cin=192, Cout=128),
         dict(S=32, D=1, B=70, Cin=128, Cout=128, prologue=_lib.PRO_AFFINE_RELU),
         dict(S=16, D=1, B=70, Cin=512, Cout=256), dict(S=16, D=1, B=70, Cin=256, prologue=_lib.PRO_AFFINE_RELU)]


@pytest.mark.parametrize('shape', REUSE)
def test_reuse_layers_move_to_the_split_input(lib, shape):
    d = desc(**shape)
    rc, ro = plan(lib, d, _lib.TC_F16, BOTH)
    assert rc == 0
    rc, flat = plan(lib, d, _lib.TC_F16, _lib.TC_PRENORM)
    assert rc == 0
    assert flat[0] == 1 and flat[3] == 0                 # without the flag: the A-reuse kernel
    assert ro[0] == 0 and ro[3] == 1                     # with it: persistent, A by TMA im2col
    assert ro[1:3] == flat[1:3]                          # the A-reuse kernel's BN and K splits
    M = d.B * d.Do * d.Ho * d.Wo
    partials = ro[2] * M * d.Cout * 4 if ro[2] > 1 else 0
    assert ws(lib, d, _lib.TC_F16, _lib.TC_PRENORM) == partials
    assert ws(lib, d, _lib.TC_F16, BOTH) == (partials + 255) // 256 * 256 + split_bytes(d)


def test_reuse_split_k_over_channel_blocks(lib):
    """K = 27 * 256 exceeds the accumulate-chain bound: two splits of two channel blocks each, as the A-reuse kernel."""
    d = desc(S=32, Cin=256, B=1)
    assert plan(lib, d, _lib.TC_F16, RO) == (0, [0, 64, 2, 1])
    assert plan(lib, d, _lib.TC_F16, 0) == (0, [1, 64, 2, 0])


# the refiner's 3-D layers on the persistent kernel: trunk conv4 (8^3) and conv5.3 (4^3)
@pytest.mark.parametrize('shape', [dict(S=8, Cin=256, Cout=256), dict(S=4, Cin=512, Cout=512)])
@pytest.mark.parametrize('pro', [_lib.PRO_NONE, _lib.PRO_AFFINE_RELU])
def test_volumes_on_the_persistent_kernel_get_the_split_input(lib, shape, pro):
    d = desc(prologue=pro, **shape)
    flags = BOTH if pro else RO
    rc, ro = plan(lib, d, _lib.TC_F16, flags)
    assert rc == 0
    assert ro[0] == 0 and ro[3] == 1
    assert plan(lib, d, _lib.TC_F16, flags & ~RO)[1] == ro[:3] + [0]     # same kernel, BN and splits
    partials = ro[2] * d.B * d.Do * d.Ho * d.Wo * d.Cout * 4 if ro[2] > 1 else 0
    assert ws(lib, d, _lib.TC_F16, flags) == (partials + 255) // 256 * 256 + split_bytes(d)


@pytest.mark.parametrize('why, d, kind, flags', [
    ('1x1', desc(S=32, k=1, pad=0), _lib.TC_F16, BOTH),
    ('stride 2', desc(S=32, stride=2), _lib.TC_F16, BOTH),
    ('tf32', desc(S=32), _lib.TC_TF32, BOTH),
    ('tf32 volume on the persistent kernel', desc(S=8, Cin=256, Cout=256), _lib.TC_TF32, BOTH),
    ('2-D plane too wide for the A-reuse kernel', desc(S=160, D=1, Cin=64), _lib.TC_F16, BOTH),
    ('prologue without prenorm', desc(S=32, prologue=_lib.PRO_AFFINE_RELU), _lib.TC_F16, RO),
    ('prologue without prenorm, persistent', desc(S=8, Cin=256, Cout=256, prologue=_lib.PRO_AFFINE), _lib.TC_F16, RO),
])
def test_reuse_im2col_is_a_noop_elsewhere(lib, why, d, kind, flags):
    rc, ro = plan(lib, d, kind, flags)
    assert rc == 0, why
    assert ro == plan(lib, d, kind, flags & ~RO)[1], why
    assert ws(lib, d, kind, flags) == ws(lib, d, kind, flags & ~RO), why


@pytest.mark.parametrize('why, fields', [
    ('lower corner -17', dict(pd=17, Do=8 + 34 - 3 + 1)),
    ('lower corner -17 in W', dict(pw=17, Wo=8 + 34 - 3 + 1)),
    ('kernel of 17 taps in D', dict(kd=17, pd=8, Do=8)),
])
def test_rank5_corner_range_falls_back(lib, why, fields):
    """The driver takes rank-5 box corners in [-16, 15] only: such a volume keeps the producer warps."""
    d = desc(S=8, Cin=256, Cout=256)
    for name, v in fields.items():
        setattr(d, name, v)
    rc, ro = plan(lib, d, _lib.TC_F16, RO)
    assert rc == 0, why
    assert ro[3] == 0, why
    assert ro == plan(lib, d, _lib.TC_F16, 0)[1], why
    assert ws(lib, d, _lib.TC_F16, RO) == ws(lib, d, _lib.TC_F16, 0), why


def test_rank5_corner_range_edge_is_taken(lib):
    d = desc(S=8, Cin=256, Cout=256)
    d.pd, d.Do = 16, 8 + 32 - 3 + 1                      # lower corner -16, upper 14
    assert plan(lib, d, _lib.TC_F16, RO)[1][3] == 1


@pytest.mark.parametrize('flags', [RO, BOTH])
def test_reuse_im2col_rejects_bad_descriptors(lib, flags):
    d = desc()
    d.out_coff = 8
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'output channel slice out of row' in lib.g6d_last_error()
    assert ws(lib, d, _lib.TC_F16, flags) == -1
    d = desc(Cin=96)
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'Cin (96) must be a multiple of 64' in lib.g6d_last_error()
    d = desc()
    d.in_coff = 64
    assert plan(lib, d, _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'input channel slice out of row' in lib.g6d_last_error()


@pytest.mark.parametrize('flags', [2, 8, RO | 2, BOTH | 16])
def test_unknown_flag_bits_rejected(lib, flags):
    assert plan(lib, desc(), _lib.TC_F16, flags)[0] == G6D_EINVAL
    assert b'bad flags' in lib.g6d_last_error()
    assert ws(lib, desc(), _lib.TC_F16, flags) == -1
