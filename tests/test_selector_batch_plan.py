"""plan_rows without a GPU: a selector layer over Q queries' rows, planned for one query's rows, gets the K splits of the
call over one query (so every query's output sums the same chains), on both tensor-core kernels and the FFMA path;
plan_rows = 0 keeps the plans the library made before the field existed."""
import ctypes

import pytest

from gen6d_b200 import _lib
from gen6d_b200.network.params import SEL_TOWERS, SEL_TOWER_POST
from gen6d_b200.network.selector import FEAT_PAD

RFN, AN, Q = 64, 5, 10                 # bench.py's reference set and batch
S = RFN * AN
TC_FLAGS = _lib.TC_PRENORM | _lib.TC_REUSE_IM2COL | _lib.TC_FOLD_SPLITS


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def desc(B, HW, cin, cout, k, prologue=_lib.PRO_NONE, group_rows=1, plan_rows=0):
    p = k // 2
    return _lib.ConvDesc(B=B, D=1, H=HW, W=HW, Cin=cin, in_cstride=cin, in_coff=0, Cout=cout, kd=1, kh=k, kw=k, stride=1,
                         pd=0, ph=p, pw=p, Do=1, Ho=HW, Wo=HW, out_cstride=cout, out_coff=0, prologue=prologue,
                         group_rows=group_rows, act=0, max_chain_k=0, plan_rows=plan_rows)


def tower_layers():
    """(name, images per query, map size, Cin, Cout, prologue) of every tower layer that runs once over all queries."""
    out = []
    for lvl, convs in enumerate(SEL_TOWERS):
        hw, pro = 16 >> lvl, None
        for i, (slot, (cin, cout)) in enumerate(sorted(convs.items())):
            post = SEL_TOWER_POST[lvl][slot]
            if i > 0:                   # the first layer forms q (.) ref: one call per query
                out.append((f'tower{lvl}.{slot}', S, hw, cin, cout, pro))
            pro = _lib.PRO_AFFINE_RELU if 'r' in post else _lib.PRO_AFFINE
            hw = hw // 2 if 'p' in post else hw
    return out


# (name, rows per query, Cin, Cout): the 1x1 layers after the towers, as [rows, 1, 1, Cin] images
ONE_BY_ONE = [('cf0', S * 16, 768, 512), ('cf3', S, 512, 512), ('sp0', S, FEAT_PAD, 512), ('sp2', S, 512, 512),
              ('att', RFN, 512, 512), ('m0', RFN, 1024, 512), ('m3', RFN, 512, 512), ('score0', RFN, 512, 512),
              ('score1', RFN, 512, 1), ('angle0', RFN, AN * FEAT_PAD, 512), ('angle1', RFN, 512, 512),
              ('angle2', RFN, 512, 1)]


def tc_plan(lib, d, kind):
    out = (ctypes.c_int * 6)(*([-7] * 6))
    rc = lib.g6d_conv_tc_plan_v2(ctypes.byref(d), kind, TC_FLAGS, out, 6)
    assert rc == 0, lib.g6d_last_error()
    return list(out)


def ffma_splits(lib, d):
    ws = lib.g6d_conv_workspace_bytes(ctypes.byref(d))
    assert ws >= 0, lib.g6d_last_error()
    M = d.B * d.Do * d.Ho * d.Wo
    return ws // (M * d.Cout * 4) if ws else 1


def layers():
    for name, n, hw, cin, cout, pro in tower_layers():
        yield name, (lambda Qn, plan, n=n, hw=hw, cin=cin, cout=cout, pro=pro:
                     desc(Qn * n, hw, cin, cout, 3, pro, group_rows=n, plan_rows=plan and plan * hw * hw))
    for name, n, cin, cout in ONE_BY_ONE:
        yield name, (lambda Qn, plan, n=n, cin=cin, cout=cout: desc(Qn * n, 1, cin, cout, 1, plan_rows=plan))


LAYERS = list(layers())


@pytest.mark.parametrize('name, make', LAYERS, ids=[n for n, _ in LAYERS])
def test_plan_rows_gives_the_per_query_splits(lib, name, make):
    one = make(1, 0)
    per_query_images = one.B
    batched = make(Q, per_query_images)
    kinds = [k for k in (_lib.TC_F16, _lib.TC_TF32) if lib.g6d_conv_tc_supported(ctypes.byref(one), k)]
    for kind in kinds:
        ref = tc_plan(lib, one, kind)
        got = tc_plan(lib, batched, kind)
        assert got[:4] == ref[:4], (name, kind, got, ref)             # kernel, BN, K splits, split input
    assert ffma_splits(lib, batched) == ffma_splits(lib, one), name
    if name in ('sp0', 'angle0', 'score1', 'angle2'):
        assert not kinds, name                                          # these run on the FFMA path


def test_plan_rows_changes_what_fills_the_gpu(lib):
    """The point of plan_rows: cf3 (1x1 512 -> 512) splits K at one query's 320 rows, which fill 12 CTAs, and not at
    ten queries' rows, which fill 100."""
    b = dict(B=Q * S, HW=1, cin=512, cout=512, k=1)
    own, planned = tc_plan(lib, desc(**b), _lib.TC_F16), tc_plan(lib, desc(**b, plan_rows=S), _lib.TC_F16)
    one = tc_plan(lib, desc(**dict(b, B=S)), _lib.TC_F16)
    assert planned[2] == one[2] > own[2]


# What the library planned before plan_rows existed, for every layer above over one query and over ten (no plan_rows):
# (fp16 plan, tf32 plan, FFMA splits), a plan being (A-reuse kernel, BN, K splits, split input, fold, x reuse) and _
# where the tensor-core path does not take the layer.
_ = None
RECORDED = {
    ('tower0.4', 1): ((0, 64, 1, 1, 0, 1), (1, 64, 1, 0, 0, 0), 1),
    ('tower0.7', 1): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower0.10', 1): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower0.13', 1): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 4),
    ('tower0.16', 1): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 4),
    ('tower1.4', 1): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower1.7', 1): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 4),
    ('tower1.10', 1): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 4),
    ('tower2.4', 1): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 4),
    ('cf0', 1): ((0, 128, 1, 0, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('cf3', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('sp0', 1): (_, _, 4),
    ('sp2', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('att', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('m0', 1): ((0, 128, 4, 0, 0, 0), (0, 128, 4, 0, 0, 0), 8),
    ('m3', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('score0', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('score1', 1): (_, _, 4),
    ('angle0', 1): (_, _, 18),
    ('angle1', 1): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('angle2', 1): (_, _, 4),
    ('tower0.4', 10): ((0, 64, 1, 1, 0, 1), (1, 64, 1, 0, 0, 0), 1),
    ('tower0.7', 10): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower0.10', 10): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower0.13', 10): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower0.16', 10): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 1),
    ('tower1.4', 10): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower1.7', 10): ((0, 128, 1, 1, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('tower1.10', 10): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 1),
    ('tower2.4', 10): ((0, 128, 2, 1, 1, 0), (0, 128, 2, 0, 0, 0), 1),
    ('cf0', 10): ((0, 128, 1, 0, 0, 0), (0, 128, 1, 0, 0, 0), 1),
    ('cf3', 10): ((0, 128, 1, 0, 0, 0), (0, 128, 1, 0, 0, 0), 3),
    ('sp0', 10): (_, _, 3),
    ('sp2', 10): ((0, 128, 1, 0, 0, 0), (0, 128, 1, 0, 0, 0), 3),
    ('att', 10): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('m0', 10): ((0, 128, 4, 0, 0, 0), (0, 128, 4, 0, 0, 0), 8),
    ('m3', 10): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('score0', 10): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('score1', 10): (_, _, 4),
    ('angle0', 10): (_, _, 14),
    ('angle1', 10): ((0, 128, 2, 0, 0, 0), (0, 128, 2, 0, 0, 0), 4),
    ('angle2', 10): (_, _, 4),
}


@pytest.mark.parametrize('name, qn', list(RECORDED), ids=[f'{n}-q{q}' for n, q in RECORDED])
def test_plan_rows_zero_keeps_the_recorded_plans(lib, name, qn):
    d = dict(LAYERS)[name](qn, 0)
    f16, tf32, ffma = RECORDED[name, qn]
    for kind, want in ((_lib.TC_F16, f16), (_lib.TC_TF32, tf32)):
        supported = bool(lib.g6d_conv_tc_supported(ctypes.byref(d), kind))
        assert supported == (want is not None), (name, kind)
        if supported:
            assert tuple(tc_plan(lib, d, kind)) == want, (name, qn, kind)
    assert ffma_splits(lib, d) == ffma, (name, qn)


def test_plan_rows_must_be_whole_images(lib):
    d = desc(Q * S, 8, 128, 128, 3, plan_rows=S * 64 + 1)
    assert lib.g6d_conv_tc_workspace_bytes(ctypes.byref(d), _lib.TC_F16) == -1
    assert b'plan_rows' in lib.g6d_last_error()
    assert lib.g6d_conv_workspace_bytes(ctypes.byref(d)) == -1
    assert b'plan_rows' in lib.g6d_last_error()
