"""Every convolution kernel and plan feature against the fp64 reference of conv_fp64_ref.py, element by element.

Each case names the instantiation it is meant to reach and asserts the exact plan (use_flat, BN, splits, split_in,
fold, xr) through g6d_conv_tc_plan_v2 before it runs, so a planner change fails here instead of silently testing
something else.  After each call the tensor-core timeout record must be clean.  The output lands in a NaN-filled buffer
(a wider row when the case writes a channel slice) and every byte outside the real outputs must still be NaN; an
input channel slice is read from a row whose other channels are NaN, so a kernel that reads them fails (a).

The matrix covers the persistent kernel conv_tc2_kernel<BN, KIND, FOLD, XR> (both operand kinds at BN 32, 64 and 128,
A gathered by the producer warps or loaded by TMA im2col from the split input: rank 4, rank 5 through reuse_im2col,
with each prologue through prenorm; folded K splits at every BN; one A box per row of taps, folded and not), the A-reuse
kernel conv_tcflat<BN, KIND> with K splits and moments, every split-K epilogue (conv_tc_reduce_kernel,
conv_tc_reduce4_kernel<2, 3, 4, 8, 0> with and without 16-byte stores, conv_tc_reduce_stats_kernel), the fused moments
of every path (epilogue, reduce, A-reuse, A-reuse order, fold) checked against the fp64 moments of the kernel's own y,
and the FFMA kernels (conv_ffma_kernel<2, 4, 8> with and without split-K, the first VGG layer alone and fused with ReLU
and max-pool, linear_smallm).  Each call runs under torch.profiler, and every kernel the case's plan predicts (see
launched: moments the convolution cannot fuse count as the separate pass that takes them) must be among the kernels it
launched; test_coverage compares those with every instantiation the planner can reach.

Operands are signed (random weights of both signs), so (b) separates an fp32-faithful result from one with a single
fp16 / TF32 rounding; the negative controls show that (b) rejects a weight without its lo half and that (a) rejects
exactly the outputs whose receptive field holds one changed input pixel.  The production replay checks sampled rows of
every convolution of one recorded predict_batch with its real operands; its correlation layers multiply post-ReLU
features by post-ReLU kernels (same-sign products, coherent sums), where (b) does not separate the classes: those keep
(a) only, and the signed matrix cases carry (b) for the same kernels and plans (row of taps, chain-bounded splits).

Measured on an H100 SXM (80 GB, 700 W): the whole file in about 22 s, the replay in about 4 s of it.
"""
import ctypes
import inspect
import os
import re
import sys
import time
from dataclasses import dataclass, field
from typing import Optional

import pytest
import torch

import conv_fp64_ref as R

pytestmark = pytest.mark.gpu

RO, PN, FO = 4, 1, 32          # _lib.TC_REUSE_IM2COL, TC_PRENORM, TC_FOLD_SPLITS
F16, TF32 = R.TC_F16, R.TC_TF32


@pytest.fixture(scope='module')
def ops():
    from gen6d_b200 import ops
    ops.require_cuda()
    return ops


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    monkeypatch.delenv('G6D_CONV_PATH', raising=False)
    monkeypatch.delenv('G6D_CONV_KIND', raising=False)


@dataclass
class Case:
    id: str
    shape: tuple                 # input (B, H, W) or (B, D, H, W), channels excluded
    cin: int
    cout: int
    k: tuple                     # (kd, kh, kw)
    plan: Optional[tuple]        # (use_flat, BN, splits, split_in, fold, xr); None: the FFMA path
    stride: int = 1
    pad: Optional[tuple] = None  # default k // 2
    kind: int = F16
    flags: int = 0
    pro: int = R.PRO_NONE
    group_rows: int = 1
    act: int = R.ACT_RELU
    bias: bool = True
    mck: int = 0                 # max_chain_k
    in_slice: Optional[tuple] = None    # (in_coff, in_cstride)
    out_slice: Optional[tuple] = None   # (out_coff, out_cstride)
    stats: Optional[int] = None  # stats_rows
    relu_x: bool = False         # post-ReLU input (still signed products: the weights have both signs)
    reaches: tuple = field(default_factory=tuple)   # what the case is meant to reach (documentation)

    def padding(self):
        return self.pad if self.pad is not None else tuple(kk // 2 for kk in self.k)


C = Case
CASES = [
    # ---- persistent kernel, A gathered by the producer warps
    C('persist-tf32-bn32-gather-m1', (681, 5, 5), 64, 24, (1, 3, 3), (0, 32, 1, 0, 0, 0), kind=TF32,
      reaches=('5x5 planes too small for the A-reuse kernel', 'M % 128 = 1', 'Cout 24 < BN')),
    C('persist-tf32-bn64-stride2-3d', (2, 9, 10, 11), 32, 40, (3, 3, 3), (0, 64, 3, 0, 0, 0), stride=2, kind=TF32,
      act=R.ACT_LEAKY01, reaches=('stride 2 in 3-D', 'leaky ReLU')),
    C('persist-tf32-bn128-1x1-m1', (1, 3, 43), 96, 136, (1, 1, 1), (0, 128, 1, 0, 0, 0), kind=TF32, act=R.ACT_NONE,
      reaches=('1x1', 'M = 129', 'two N tiles, the second 8 wide')),
    C('persist-f16-bn32-stride2', (16, 65, 63), 64, 32, (1, 3, 3), (0, 32, 1, 0, 0, 0), stride=2, bias=False,
      reaches=('f16 gather', 'no bias')),
    C('persist-f16-bn64-3d-affine-relu', (3, 5, 6, 7), 128, 56, (3, 3, 3), (0, 64, 11, 0, 0, 0), pro=R.PRO_AFFINE_RELU,
      group_rows=2, reaches=('prologue in the producers (no prenorm)', 'tiles across volumes', 'Cout 56')),
    C('persist-f16-bn128-1x1-corr', (4, 6, 6), 128, 130, (1, 1, 1), (0, 128, 1, 0, 0, 0), pro=R.PRO_CORR, group_rows=4,
      act=R.ACT_NONE, reaches=('per-position prologue, 1x1', 'Cout 130')),
    C('persist-f16-bn64-valid', (9, 9, 10), 64, 64, (1, 3, 3), (0, 64, 2, 1, 0, 0), pad=(0, 0, 0),
      reaches=('valid 3x3, rank-4 im2col', 'M = 7 * 8 * 9')),
    # ---- persistent kernel, A by TMA im2col (rank 4 from the split input, rank 5 through reuse_im2col)
    C('persist-f16-bn128-im2col-m1', (681, 5, 5), 128, 200, (1, 3, 3), (0, 128, 1, 1, 0, 0),
      reaches=('rank-4 im2col', 'M % 128 = 1', 'Cout 200: second N tile partial')),
    C('persist-f16-bn32-im2col-inslice', (9, 7, 7), 64, 20, (1, 3, 3), (0, 32, 2, 1, 0, 0), in_slice=(8, 80),
      reaches=('input channel slice [8, 72) of 80, NaN elsewhere', 'Cout 20')),
    C('prenorm-affine', (20, 6, 6), 64, 64, (1, 3, 3), (0, 64, 2, 1, 0, 0), flags=PN, pro=R.PRO_AFFINE, group_rows=4,
      reaches=('split pass applies G6D_PRO_AFFINE', 'groups of 4 items')),
    C('prenorm-affine-relu-bn32', (33, 4, 4), 64, 32, (1, 3, 3), (0, 32, 2, 1, 0, 0), flags=PN, pro=R.PRO_AFFINE_RELU,
      group_rows=1, act=R.ACT_LEAKY01, reaches=('split pass applies G6D_PRO_AFFINE_RELU', 'M = 528')),
    C('prenorm-corr', (12, 8, 8), 128, 64, (1, 3, 3), (0, 64, 4, 1, 0, 0), flags=PN, pro=R.PRO_CORR, group_rows=12,
      reaches=('split pass applies G6D_PRO_CORR, group_rows = S',)),
    C('rank5-volume', (2, 6, 7, 9), 64, 48, (3, 3, 3), (0, 64, 6, 1, 0, 0), flags=RO,
      reaches=('rank-5 im2col', 'tiles across z-planes and volumes')),
    C('rank5-d1-kd3', (3, 1, 9, 10), 64, 64, (3, 3, 3), (0, 64, 1, 1, 0, 1), flags=RO,
      reaches=('rank-5 im2col of a single plane with kd = 3: the z taps are all padding but one',)),
    C('rank5-prenorm-affine-relu', (2, 4, 5, 6), 128, 96, (3, 3, 3), (0, 128, 11, 1, 0, 0), flags=RO | PN,
      pro=R.PRO_AFFINE_RELU, group_rows=1, reaches=('rank-5 im2col with the prologue in the split pass',)),
    # ---- folded K splits (one CTA sums a tile's splits)
    C('fold-bn128-m127', (1, 81, 207), 256, 128, (1, 3, 3), (0, 128, 2, 1, 1, 0), flags=FO,
      reaches=('FOLD at BN 128', 'chain-bounded splits (K 2304 > 2048)', 'M % 128 = 127', 'plane too wide for A-reuse')),
    C('fold-bn64-mck', (1, 81, 207), 128, 48, (1, 3, 3), (0, 64, 3, 1, 1, 0), flags=FO, mck=128,
      reaches=('FOLD at BN 64', 'splits from max_chain_k')),
    C('fold-bn32-mck-m127', (1, 81, 207), 128, 32, (1, 3, 3), (0, 32, 3, 1, 1, 0), flags=FO, mck=64, act=R.ACT_NONE,
      reaches=('FOLD at BN 32', 'M % 128 = 127')),
    C('fold-bn32-stats', (262, 8, 8), 128, 32, (1, 3, 3), (0, 32, 3, 1, 1, 0), flags=FO, mck=64, stats=64,
      reaches=('FOLD with fused moments per 8x8 plane: fold_moments_kernel', '131 tiles')),
    # ---- one A box per row of taps (BN 64, the A-reuse kernel's K order)
    C('xr-unfolded', (3, 13, 13), 64, 64, (1, 3, 3), (0, 64, 1, 1, 0, 1), flags=RO, out_slice=(40, 136),
      reaches=('XR', 'tiles span planes and images', 'output slice [40, 104) of 136')),
    C('xr-folded', (66, 16, 16), 256, 64, (1, 3, 3), (0, 64, 2, 1, 1, 1), flags=RO | FO, mck=384,
      reaches=('XR + FOLD',)),
    C('xr-1x7-splits', (2, 12, 40), 256, 50, (1, 1, 7), (0, 64, 4, 1, 0, 1), flags=RO, pad=(0, 0, 3),
      reaches=('XR with a row of 7 taps', 'unfolded splits, Cout 50: conv_tc_reduce_kernel')),
    # ---- the A-reuse kernel
    C('flat-tf32-bn32', (3, 20, 21), 64, 32, (1, 3, 3), (1, 32, 2, 0, 0, 0), kind=TF32, reaches=('conv_tcflat<32, TF32>',)),
    C('flat-tf32-bn64', (3, 20, 21), 64, 64, (1, 3, 3), (1, 64, 2, 0, 0, 0), kind=TF32, act=R.ACT_NONE,
      reaches=('conv_tcflat<64, TF32>',)),
    C('flat-tf32-bn128-m16', (2, 40, 45), 64, 96, (1, 3, 3), (1, 128, 2, 0, 0, 0), kind=TF32,
      reaches=('conv_tcflat<128, TF32>', 'Cout 96')),
    C('flat-f16-bn32-stats', (4, 24, 24), 64, 24, (1, 3, 3), (1, 32, 1, 0, 0, 0), stats=576, act=R.ACT_NONE,
      reaches=('conv_tcflat<32, F16>', 'moments in the A-reuse epilogue')),
    C('flat-f16-bn64-3d-splits', (1, 7, 37, 47), 128, 48, (1, 3, 3), (1, 64, 2, 0, 0, 0), pad=(0, 1, 1),
      reaches=('conv_tcflat<64, F16> on a 1x3x3 volume layer', 'K splits over channel blocks', 'M % 128 = 13')),
    C('flat-f16-bn128-slices', (2, 40, 45), 64, 96, (1, 3, 3), (1, 128, 1, 0, 0, 0), in_slice=(4, 72),
      out_slice=(3, 101), reaches=('conv_tcflat<128, F16>', 'input slice [4, 68) of 72', 'odd output slice')),
    C('flat-f16-bn64-splits-stats', (2, 20, 24), 512, 64, (1, 3, 3), (1, 64, 8, 0, 0, 0), stats=480,
      reaches=('A-reuse with splits: conv_tc_reduce_stats_kernel',)),
    C('ro-moments', (2, 16, 16, 16), 64, 64, (3, 3, 3), (0, 64, 1, 1, 0, 1), flags=RO, stats=4096, act=R.ACT_NONE,
      reaches=('A-reuse K order, one split: flat_moments_kernel',)),
    # ---- split-K epilogues
    C('reduce4-s2-vec', (1, 33, 128), 512, 256, (1, 1, 1), (0, 128, 2, 0, 0, 0), act=R.ACT_NONE, reaches=('conv_tc_reduce4_kernel<2>',)),
    C('reduce4-s3-scalar', (1, 22, 128), 768, 256, (1, 1, 1), (0, 128, 3, 0, 0, 0), out_slice=(1, 259),
      reaches=('conv_tc_reduce4_kernel<3>, scalar stores (odd out_coff)',)),
    C('reduce4-s4-vec', (1, 33, 128), 1024, 128, (1, 1, 1), (0, 128, 4, 0, 0, 0), act=R.ACT_LEAKY01, reaches=('conv_tc_reduce4_kernel<4>',)),
    C('reduce4-s8-scalar', (2, 8, 8), 2048, 128, (1, 1, 1), (0, 128, 8, 0, 0, 0), out_slice=(5, 135), kind=TF32,
      reaches=('conv_tc_reduce4_kernel<8>, scalar stores',)),
    C('reduce4-s0-vec', (1, 20, 128), 1536, 128, (1, 1, 1), (0, 128, 6, 0, 0, 0), reaches=('conv_tc_reduce4_kernel<0> (5 or 6 splits)',)),
    C('reduce4-s2-scalar', (1, 33, 128), 512, 256, (1, 1, 1), (0, 128, 2, 0, 0, 0), out_slice=(3, 259),
      reaches=('conv_tc_reduce4_kernel<2>, scalar stores',)),
    C('reduce4-s4-scalar', (1, 33, 128), 1024, 128, (1, 1, 1), (0, 128, 4, 0, 0, 0), out_slice=(1, 133),
      reaches=('conv_tc_reduce4_kernel<4>, scalar stores',)),
    C('reduce4-s8-vec', (2, 8, 8), 2048, 128, (1, 1, 1), (0, 128, 8, 0, 0, 0), kind=TF32, reaches=('conv_tc_reduce4_kernel<8>',)),
    C('reduce4-s0-scalar', (1, 20, 128), 1536, 128, (1, 1, 1), (0, 128, 6, 0, 0, 0), out_slice=(7, 137), act=R.ACT_NONE,
      reaches=('conv_tc_reduce4_kernel<0>, scalar stores',)),
    C('reduce-stats', (2, 8, 8), 1024, 64, (1, 1, 1), (0, 64, 4, 0, 0, 0), stats=64, act=R.ACT_NONE,
      reaches=('conv_tc_reduce_stats_kernel',)),
    C('reduce-cout-odd', (1, 2, 3, 5), 512, 18, (3, 3, 3), (0, 32, 54, 0, 0, 0), stride=2, kind=TF32, out_slice=(2, 23),
      reaches=('conv_tc_reduce_kernel (Cout % 4 = 2)', 'stride 2 in 3-D with splits')),
    C('epilogue-stats', (6, 8, 8), 128, 64, (1, 1, 1), (0, 64, 1, 0, 0, 0), stats=32,
      reaches=('moments in the persistent epilogue, 32-row groups',)),
]
CASE_IDS = [c.id for c in CASES]


def desc_of(x, c, ocs, oco, in_coff):
    from gen6d_b200 import _lib
    if x.dim() == 4:
        (B, H, W, cs), D = x.shape, 1
    else:
        B, D, H, W, cs = x.shape
    (kd, kh, kw), (pd, ph, pw), s = c.k, c.padding(), c.stride
    return _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=c.cin, in_cstride=cs, in_coff=in_coff, Cout=c.cout, kd=kd, kh=kh, kw=kw,
                         stride=s, pd=pd, ph=ph, pw=pw, Do=(D + 2 * pd - kd) // s + 1, Ho=(H + 2 * ph - kh) // s + 1,
                         Wo=(W + 2 * pw - kw) // s + 1, out_cstride=ocs, out_coff=oco, prologue=c.pro,
                         group_rows=c.group_rows, act=c.act, max_chain_k=c.mck)


def plan_of(d, kind, flags):
    from gen6d_b200 import _lib
    out = (ctypes.c_int * 6)()
    _lib.check(_lib.lib().g6d_conv_tc_plan_v2(ctypes.byref(d), kind, flags, out, 6), 'g6d_conv_tc_plan_v2')
    return tuple(out)


def debug_record():
    from gen6d_b200 import _lib
    rec = (ctypes.c_int * 8)()
    _lib.check(_lib.lib().g6d_conv_tc_debug(rec), 'g6d_conv_tc_debug')
    return list(rec)


def launched(d, kind, flags, plan, stats):
    """The kernels one tensor-core call of this plan launches, as g6d_conv_tc_ex and its dispatch choose them.  stats:
    the stats_rows of the call; moments the convolution cannot fuse (g6d_conv_tc_stats_supported) are taken by
    instnorm_partial, a pass of its own, and count as that."""
    from gen6d_b200 import _lib
    if stats and not _lib.lib().g6d_conv_tc_stats_supported(ctypes.byref(d), kind, stats):
        stats, unfused = None, {'in_stats_partial_kernel (unfused moments)'}
    else:
        unfused = set()
    use_flat, bn, splits, split_in, fold, xr = plan
    k = 'F16' if kind == F16 else 'TF32'
    reuse_order = not use_flat and split_in and plan_of(d, kind, flags & ~RO)[0] == 1
    out = set()
    if use_flat:
        out.add(f'conv_tcflat_kernel<{bn}, {k}>')
    else:
        out.add(f'conv_tc2_kernel<{bn}, {k}, {"true" if fold else "false"}, {"true" if xr else "false"}>')
    if split_in:
        rank5 = d.D > 1 or d.kd > 1
        out.add(f'split_input_f16_kernel rank {5 if rank5 else 4}' + (f' prologue {d.prologue}' if d.prologue else ''))
    if stats:
        if reuse_order and splits == 1:
            out.add('flat_moments_kernel')
        elif fold:
            out.add('fold_moments_kernel')
        elif splits > 1:
            out.add('conv_tc_reduce_stats_kernel')
        else:
            out.add('A-reuse epilogue moments' if use_flat else 'persistent epilogue moments')
    elif splits > 1 and not fold:
        if d.Cout % 4:
            out.add('conv_tc_reduce_kernel')
        else:
            vec = d.out_cstride % 4 == 0 and d.out_coff % 4 == 0
            out.add(f'conv_tc_reduce4_kernel<{splits if splits in (2, 3, 4, 8) else 0}> {"vec" if vec else "scalar"}')
    return out | unfused


def profiled(fn):
    """(fn(), the names of the GPU kernels it launched, as torch.profiler records them)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch.cuda.synchronize()
    return r, {e.name for e in prof.events()}


KIND_ARG = {'F16': str(F16), 'TF32': str(TF32)}


def ran(key, names):
    """Whether the kernel of a launched() entry ('name<template args> notes') is among the profiled kernel names, with
    the same template arguments when the entry gives them.  Entries that are no kernel of their own (moments in a
    convolution's epilogue) return None."""
    m = re.match(r'(\w+)(?:<([^>]*)>)?', key)
    base, targs = m.group(1), m.group(2)
    if not base.endswith('_kernel'):
        return None
    want = None if targs is None else [KIND_ARG.get(t.strip(), t.strip()) for t in targs.split(',')]
    for n in names:
        for hit in re.finditer(r'\b' + base + r'\b(?:<([^>]*)>)?', n):
            got = [re.sub(r'^\(\w+\)', '', t.strip()) for t in (hit.group(1) or '').split(',')]
            if want is None or got == want:
                return True
    return False


def verify_launches(cid, modeled, names):
    """Asserts that every kernel launched() predicts ran, and returns the entries the coverage test may count."""
    missing = [k for k in modeled if ran(k, names) is False]
    assert not missing, f'{cid}: predicted kernels {missing} did not run; the profiler saw {sorted(names)}'
    return set(modeled)


def operands(c, seed, dev='cuda'):
    """(x with NaN outside the input slice, w, bias, pro_scale, pro_shift, in_coff)"""
    gen = torch.Generator().manual_seed(seed)
    in_coff, ics = c.in_slice or (0, c.cin)
    x = torch.full((*c.shape, ics), float('nan'))
    v = torch.randn(*c.shape, c.cin, generator=gen) + (0.0 if c.relu_x else 0.25)
    x[..., in_coff:in_coff + c.cin] = v.clamp_min(0) if c.relu_x else v
    taps = c.k[0] * c.k[1] * c.k[2]
    w = torch.randn(c.cout, c.cin, *c.k, generator=gen) * (2 / (taps * c.cin)) ** .5
    b = torch.randn(c.cout, generator=gen) * 0.5 if c.bias else None
    ps = pb = None
    B = c.shape[0]
    plane = 1
    for n in c.shape[1:]:
        plane *= n
    if c.pro == R.PRO_CORR:
        ps, pb = torch.rand(plane, c.cin, generator=gen) + 0.5, torch.randn(c.cin, generator=gen) * 0.2
    elif c.pro != R.PRO_NONE:
        groups = (B - 1) // c.group_rows + 1
        ps, pb = torch.rand(groups, c.cin, generator=gen) + 0.5, torch.randn(groups, c.cin, generator=gen) * 0.5
    cu = lambda t: None if t is None else t.to(dev).contiguous()
    return cu(x), cu(w), cu(b), cu(ps), cu(pb), in_coff


ASSERTED = {}       # case id -> (plan, kernels launched)


def run_tc_case(ops, c, monkeypatch, x, w, b, ps, pb, in_coff, w_lo_zero=False):
    """Packs, plans, runs and returns (y [M, Cout] of the real outputs, stats or None, plan)."""
    monkeypatch.setenv('G6D_CONV_KIND', 'f16' if c.kind == F16 else 'tf32')
    pc = ops.pack_conv(w, b, stride=c.stride, pad=c.padding())
    assert pc.kind == c.kind and pc.w_hi is not None
    pc.max_chain_k = c.mck
    if w_lo_zero:
        pc.w_lo.zero_()
    oco, ocs = c.out_slice or (0, c.cout)
    d = desc_of(x, c, ocs, oco, in_coff)
    plan = plan_of(d, c.kind, c.flags)
    if c.plan is not None:
        assert plan == c.plan, f'{c.id}: plan {plan}, the case was written for {c.plan}'
    out_shape = (*x.shape[:1], *(n for n in (d.Do, d.Ho, d.Wo)[(0 if x.dim() == 5 else 1):]), ocs)
    out = torch.full(out_shape, float('nan'), device='cuda')
    assert debug_record()[0] == 0
    r, names = profiled(lambda: ops.conv(
        x, pc, prologue=c.pro, pro_scale=ps, pro_shift=pb, group_rows=c.group_rows, act=c.act, in_coff=in_coff, out=out,
        out_coff=oco, stats_rows=c.stats, prenorm=bool(c.flags & PN), reuse_im2col=bool(c.flags & RO),
        fold_splits=bool(c.flags & FO)))
    ASSERTED[c.id] = (plan, verify_launches(c.id, launched(d, c.kind, c.flags, plan, c.stats), names))
    rec = debug_record()
    assert rec[0] == 0, f'{c.id}: tensor-core pipeline timeout {rec}'
    flat = out.reshape(-1, ocs)
    assert bool(torch.isnan(flat[:, :oco]).all()) and bool(torch.isnan(flat[:, oco + c.cout:]).all()), \
        f'{c.id}: bytes outside the output slice were written'
    return flat[:, oco:oco + c.cout], (r[1] if c.stats else None), plan


def reference_of(c, x, w, b, ps, pb, in_coff):
    return R.reference(x, w, b, stride=c.stride, pad=c.padding(), prologue=c.pro, scale=ps, shift=pb,
                       group_rows=c.group_rows, act=c.act, in_coff=in_coff)


@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_conv_tc_case(ops, monkeypatch, c):
    x, w, b, ps, pb, in_coff = operands(c, seed=CASE_IDS.index(c.id) + 100)
    y, st, plan = run_tc_case(ops, c, monkeypatch, x, w, b, ps, pb, in_coff)
    print(f'\n{c.id}: plan (use_flat, BN, splits, split_in, fold, xr) = {plan}; '
          f'{sorted(ASSERTED[c.id][1])}')
    assert not bool(torch.isnan(y).any()), f'{c.id}: NaN in the output (a channel outside the input slice was read?)'
    ref, mag, s = reference_of(c, x, w, b, ps, pb, in_coff)
    R.check(c.id, y, ref, mag, s)
    if c.stats:
        R.check_moments(c.id, st, y, c.stats)


# ---------------------------------------------------------------------------------------------------- FFMA path
FFMA_CASES = [
    C('ffma-tn2', (3, 11, 13), 12, 20, (1, 3, 3), None, bias=False, in_slice=(4, 20), out_slice=(1, 23),
      reaches=('conv_ffma_kernel<2>', 'no split', 'input and output slices')),
    C('ffma-tn4-splitk', (1, 4, 5), 256, 40, (1, 3, 3), None, act=R.ACT_LEAKY01,
      reaches=('conv_ffma_kernel<4> with split-K', 'conv_splitk_reduce_kernel')),
    C('ffma-tn8-affine', (5, 7, 9), 16, 130, (1, 3, 3), None, pro=R.PRO_AFFINE_RELU, group_rows=2,
      reaches=('conv_ffma_kernel<8>', 'affine + ReLU prologue')),
    C('ffma-tn8-splitk-3d', (1, 4, 4, 4), 64, 72, (3, 3, 3), None, stride=2, pro=R.PRO_CORR, act=R.ACT_NONE,
      reaches=('conv_ffma_kernel<8> with split-K', 'stride 2 in 3-D', 'per-position prologue')),
    C('ffma-head-cout3', (2, 30, 41), 64, 3, (1, 3, 3), None, act=R.ACT_NONE,
      reaches=('a head last layer: Cout < 16 never takes the tensor cores',)),
    C('ffma-first-layer', (2, 33, 30), 4, 64, (1, 3, 3), None, reaches=('conv3x3_c4_o64_kernel',)),
]


def ffma_expected(c, M, K):
    bn = 128 if c.cout > 64 else (64 if c.cout > 32 else 32)
    ctas = -(-M // 128) * -(-c.cout // bn)
    ktiles = -(-K // 16)
    splits = 1
    if ctas < 132 and ktiles >= 16:
        splits = min(64, max(1, min(-(-264 // ctas), ktiles // 8)))
        per = -(-ktiles // splits)
        splits = -(-ktiles // per)
    return {32: 2, 64: 4, 128: 8}[bn], splits


@pytest.mark.parametrize('c', FFMA_CASES, ids=[c.id for c in FFMA_CASES])
def test_conv_ffma_case(ops, monkeypatch, c):
    monkeypatch.setenv('G6D_CONV_PATH', 'ffma')
    x, w, b, ps, pb, in_coff = operands(c, seed=500 + [f.id for f in FFMA_CASES].index(c.id))
    if c.id == 'ffma-first-layer':
        x[..., 3] = 0                       # the RGB + zero channel layout the kernel is written for
    pc = ops.pack_conv(w, b, stride=c.stride, pad=c.padding())
    oco, ocs = c.out_slice or (0, c.cout)
    d = desc_of(x, c, ocs, oco, in_coff)
    M, K = d.B * d.Do * d.Ho * d.Wo, c.k[0] * c.k[1] * c.k[2] * c.cin
    first = c.cin == 4 and c.cout == 64 and c.k == (1, 3, 3) and c.stride == 1 and not c.pro and ocs == 64 and x.dim() == 4
    tn, splits = ffma_expected(c, M, K)
    from gen6d_b200 import _lib
    ws = _lib.lib().g6d_conv_workspace_bytes(ctypes.byref(d))
    assert ws == (splits * M * c.cout * 4 if splits > 1 else 0), (ws, splits)
    what = 'conv3x3_c4_o64_kernel' if first else f'conv_ffma_kernel<{tn}>' + (f' + conv_splitk_reduce_kernel ({splits} splits)'
                                                                             if splits > 1 else '')
    print(f'\n{c.id}: {what}')
    out_shape = (*x.shape[:1], *(n for n in (d.Do, d.Ho, d.Wo)[(0 if x.dim() == 5 else 1):]), ocs)
    out = torch.full(out_shape, float('nan'), device='cuda')
    _, names = profiled(lambda: ops.conv(x, pc, prologue=c.pro, pro_scale=ps, pro_shift=pb, group_rows=c.group_rows,
                                         act=c.act, in_coff=in_coff, out=out, out_coff=oco))
    modeled = {what.split(' + ')[0]} | ({'conv_splitk_reduce_kernel'} if splits > 1 and not first else set())
    ASSERTED[c.id] = (None, verify_launches(c.id, modeled, names))
    flat = out.reshape(-1, ocs)
    assert bool(torch.isnan(flat[:, :oco]).all()) and bool(torch.isnan(flat[:, oco + c.cout:]).all())
    y = flat[:, oco:oco + c.cout]
    ref, mag, s = reference_of(c, x, w, b, ps, pb, in_coff)
    R.check(c.id, y, ref, mag, s, tau_b=R.TAU_B_FFMA)


@pytest.mark.parametrize('B, H, W', [(2, 30, 26), (3, 28, 34)])          # H / 2 odd and even
def test_vgg_first_block(ops, B, H, W):
    """conv3x3_c4_o64_relu_pool_kernel: max over each 2x2 window of ReLU(conv).  The pooled error is at most the largest
    error in the window, so a pooled element is held to the largest mag (a) and s (b) of its window."""
    gen = torch.Generator().manual_seed(H * W)
    x = torch.rand(B, H, W, 4, generator=gen) * 2 - 0.5
    x[..., 3] = 0
    w = torch.randn(64, 4, 3, 3, generator=gen) * (2 / 27) ** .5
    b = torch.randn(64, generator=gen) * 0.1
    pc = ops.pack_conv(w.cuda(), b.cuda(), pad=1)
    y, names = profiled(lambda: ops.vgg_first_block(x.cuda(), pc))
    ref, mag, s = R.reference(x.cuda(), w.reshape(64, 4, 1, 3, 3).cuda(), b.cuda(), pad=(0, 1, 1), act=R.ACT_RELU)
    pool = lambda t: torch.nn.functional.max_pool2d(t.reshape(B, H, W, 64).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    ref_p, mag_p, s_p = pool(ref).reshape(-1, 64), pool(mag).reshape(-1, 64), pool(s).reshape(-1, 64)
    ASSERTED[f'vgg-{H}'] = (None, verify_launches(f'vgg-{H}', {'conv3x3_c4_o64_relu_pool_kernel'}, names))
    print(f'\nvgg_first_block B={B} H={H} W={W}:')
    R.check(f'vgg_first_block {H}x{W}', y.reshape(-1, 64), ref_p, mag_p, s_p, tau_b=R.TAU_B_FFMA)


@pytest.mark.parametrize('M', [1, 5, 8])
def test_linear_smallm(ops, M):
    gen = torch.Generator().manual_seed(M)
    K, N = 2052, 67
    x = torch.randn(M, K, generator=gen).cuda()
    w = torch.randn(N, K, generator=gen).cuda() * K ** -.5
    b = torch.randn(N, generator=gen).cuda()
    for act in (R.ACT_NONE, R.ACT_LEAKY01):
        y, names = profiled(lambda: ops.linear_smallm(x, w, b, act=act))
        ref, mag, s = R.reference(x.reshape(M, 1, 1, K), w.reshape(N, K, 1, 1, 1), b, act=act)
        R.check(f'linear_smallm M={M} act={act}', y, ref, mag, s, tau_b=R.TAU_B_FFMA)
    ASSERTED[f'linear-{M}'] = (None, verify_launches(f'linear-{M}', {'linear_smallm_kernel'}, names))


# ---------------------------------------------------------------------------------------------------- negative controls
@pytest.mark.parametrize('cid', ['persist-f16-bn128-im2col-m1', 'persist-tf32-bn128-1x1-m1'])
def test_negative_control_lo_half_dropped(ops, monkeypatch, cid):
    """With the weights' lo halves zeroed only w_hi reaches the tensor cores: (b) must reject the result by at least
    8x its bound."""
    c = CASES[CASE_IDS.index(cid)]
    x, w, b, ps, pb, in_coff = operands(c, seed=CASE_IDS.index(c.id) + 100)
    y, _, _ = run_tc_case(ops, c, monkeypatch, x, w, b, ps, pb, in_coff, w_lo_zero=True)
    ref, mag, s = reference_of(c, x, w, b, ps, pb, in_coff)
    a, rb, _ = R.measure(y, ref, mag, s)
    fb = rb / R.TAU_B_TC
    print(f'\nnegative control, {cid} without w_lo: (a) {a / R.TAU_A:.3g} of tau_a, (b) rms {rb:.3e} = {fb:.3g} of tau_b')
    assert fb >= 8, f'(b) does not reject a weight without its lo half: {fb:.3g} of tau_b'


def test_negative_control_one_border_pixel(ops, monkeypatch):
    """One input pixel on the image border is changed after the kernel ran and the reference is computed from the
    changed input: (a) must fail, by at least 8x, at exactly the outputs whose receptive field holds that pixel (stride
    2, 3x3: one to four of them per channel), and hold everywhere else."""
    c = Case('neg-border', (2, 9, 11), 64, 40, (1, 3, 3), (0, 64, 2, 0, 0, 0), stride=2, act=R.ACT_NONE)
    x, w, b, ps, pb, in_coff = operands(c, seed=7)
    w = w.sign() * (w.abs() + 0.05)           # no weight near zero, so every affected output moves by > 0.05 |dx|
    y, _, _ = run_tc_case(ops, c, monkeypatch, x, w, b, ps, pb, in_coff)
    bi, yi, xi, ch = 1, 0, 6, 17              # image 1, top row, column 6, one channel
    x2 = x.clone()
    x2[bi, yi, xi, ch] += 3.0
    ref, mag, s = reference_of(c, x2, w, b, ps, pb, in_coff)
    err = (y.double() - ref).abs() / mag
    fail = err > R.TAU_A
    hit = torch.zeros(2, 1, 9, 11, dtype=torch.float64, device='cuda')
    hit[bi, 0, yi, xi] = 1
    field_ = torch.nn.functional.conv2d(hit, torch.ones(1, 1, 3, 3, dtype=torch.float64, device='cuda'), stride=2,
                                        padding=1).permute(0, 2, 3, 1).reshape(-1, 1) > 0
    want = field_.expand_as(fail)
    n = int(field_.sum())
    worst_in = float(err[want].min() / R.TAU_A)
    print(f'\nnegative control, one border pixel: {n} outputs x {c.cout} channels in its receptive field, smallest (a) '
          f'ratio there {worst_in:.3g} of tau_a; largest elsewhere {float(err[~want].max() / R.TAU_A):.3g}')
    assert 1 <= n <= 4
    assert torch.equal(fail, want), 'the elements (a) rejects are not the receptive field of the changed pixel'
    assert worst_in >= 8


# ---------------------------------------------------------------------------------------------------- production replay
def test_production_replay_sampled(ops):
    """Every convolution of one recorded predict_batch (batch 2, one refinement), replayed eagerly: each call's input and
    prologue operands are snapshotted, the call runs, and its output rows on the image (or volume) borders, the first
    and last 128-row tile and about 1024 random rows are checked against the fp64 reference of those rows with the
    call's real operands.  The weights come from fp32 the kernels never read: a layer's FFMA layout, or for the
    detector's correlation kernels (packed for the tensor cores only) the fp32 features ops.split_operand split, taken
    while the step is recorded.  Calls with coherent sums (the correlation: post-ReLU features against post-ReLU
    kernels, median |ref| / mag above R.COHERENT) keep (a) only."""
    t0 = time.time()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
    try:
        import conv_breakdown
    finally:
        sys.path.pop(0)
    sources, split = {}, ops.split_operand

    def recording_split(x, kind=None):
        hi, lo, k = split(x, kind)
        sources[hi.data_ptr()] = x.detach().clone()          # the fp32 rows the hi / lo halves were made from
        return hi, lo, k
    ops.split_operand = recording_split
    try:
        _, rec = conv_breakdown.record_step(2, 1)
    finally:
        ops.split_operand = split
    t_rec = time.time() - t0
    orig = ops.conv
    gen = torch.Generator(device='cpu').manual_seed(0)
    sig = inspect.signature(orig)
    worst, failed, n_calls = [0.0, 0.0, 0.0], [], [0, 0]

    def wrapped(*args, **kwargs):
        call = sig.bind(*args, **kwargs)
        call.apply_defaults()
        a = call.arguments
        x, pc, prologue, group_rows, act = a['x'], a['pc'], a['prologue'], a['group_rows'], a['act']
        in_coff, out_coff, stats_rows = a['in_coff'], a['out_coff'], a['stats_rows']
        xs = x.clone()                                    # the operands as the call sees them
        ps = None if a['pro_scale'] is None else a['pro_scale'].clone()
        pb = None if a['pro_shift'] is None else a['pro_shift'].clone()
        prof = ops.enable_profiling()
        try:
            r = orig(*args, **kwargs)
        finally:
            calls = ops.collect_profile(prof).get('#calls')             # also switches the profiling off again
        path = 'tc' if calls else 'ffma'                                # only tensor-core launches carry a tag
        y = r[0] if stats_rows is not None else r
        ocs = y.shape[-1]
        five = xs.unsqueeze(1) if xs.dim() == 4 else xs
        B = five.shape[0]
        Do, Ho, Wo = R.out_dims(five.shape, pc.k, pc.stride, pc.pad)
        M = B * Do * Ho * Wo
        yr = y.reshape(M, ocs)[:, out_coff:out_coff + pc.cout]
        idx = torch.arange(M)
        xo, t = idx % Wo, idx // Wo
        yo, zo = t % Ho, (t // Ho) % Do
        border = (xo == 0) | (xo == Wo - 1) | (yo == 0) | (yo == Ho - 1) | (((zo == 0) | (zo == Do - 1)) & (Do > 1))
        pick = border.clone()
        pick[:128] = True
        pick[max(0, (M - 1) // 128 * 128):] = True
        pick[torch.randint(0, M, (1024,), generator=gen)] = True
        rows = torch.nonzero(pick).flatten()
        source = None if pc.w is not None else sources[pc.w_hi.data_ptr()]
        wd = R.dense_weight(pc, source)
        ref, mag, s = R.reference_rows(xs, wd, rows, pc.bias, stride=pc.stride, pad=pc.pad, prologue=prologue, scale=ps,
                                       shift=pb, group_rows=group_rows, act=act, in_coff=in_coff)
        got = yr[rows.to(yr.device)]
        coh = R.coherence(ref, mag)
        coherent = coh > R.COHERENT
        name = (f'{path} M={M} N={pc.cout} K={pc.k[0] * pc.k[1] * pc.k[2] * pc.cin} k={pc.k} s={pc.stride} pro={prologue} '
                f'rows={rows.numel()} ({int(border.sum())} on borders){" fp32 split source" if source is not None else ""} '
                f'coherence {coh:.2f}')
        n_calls[0] += 1
        n_calls[1] += source is not None
        try:
            fa, fb = R.check(name, got, ref, mag, s, tau_b=R.TAU_B_TC if path == 'tc' else R.TAU_B_FFMA,
                             class_b=not coherent)
        except AssertionError as e:
            failed.append(str(e))
        else:
            worst[0] = max(worst[0], fa)
            worst[2 if coherent else 1] = max(worst[2 if coherent else 1], fb)
        return r

    print()
    ops.conv = wrapped
    try:
        with torch.no_grad():
            for fn, inputs in rec:
                fn(*inputs)
    finally:
        ops.conv = orig
    torch.cuda.synchronize()
    print(f'production replay: {n_calls[0]} convolutions ({n_calls[1]} with tensor-core-only weights, checked against '
          f'their fp32 source), worst (a) {worst[0]:.3g} of tau_a, worst (b) {worst[1]:.3g} of tau_b (coherent sums, not '
          f'asserted: {worst[2]:.3g}); {time.time() - t0:.1f} s in all, recording {t_rec:.1f} s')
    assert n_calls[0] > 50 and n_calls[1] > 0
    assert not failed, '\n'.join(failed)


# ---------------------------------------------------------------------------------------------------- coverage
# every kernel instantiation and launch variant make_plan and g6d_conv_tc_ex can reach, and the FFMA kernels
REACHABLE = (
    [f'conv_tc2_kernel<{bn}, {k}, false, false>' for k in ('TF32', 'F16') for bn in (32, 64, 128)]
    + [f'conv_tc2_kernel<{bn}, F16, true, false>' for bn in (32, 64, 128)]
    + ['conv_tc2_kernel<64, F16, false, true>', 'conv_tc2_kernel<64, F16, true, true>']
    + [f'conv_tcflat_kernel<{bn}, {k}>' for k in ('TF32', 'F16') for bn in (32, 64, 128)]
    + ['split_input_f16_kernel rank 4', 'split_input_f16_kernel rank 5']
    + [f'split_input_f16_kernel rank 4 prologue {p}' for p in (1, 2, 3)] + ['split_input_f16_kernel rank 5 prologue 2']
    + ['conv_tc_reduce_kernel', 'conv_tc_reduce_stats_kernel', 'flat_moments_kernel', 'fold_moments_kernel',
       'A-reuse epilogue moments', 'persistent epilogue moments']
    + [f'conv_tc_reduce4_kernel<{s}> {v}' for s in (2, 3, 4, 8, 0) for v in ('vec', 'scalar')]
    + ['conv_ffma_kernel<2>', 'conv_ffma_kernel<4>', 'conv_ffma_kernel<8>', 'conv_splitk_reduce_kernel',
       'conv3x3_c4_o64_kernel', 'conv3x3_c4_o64_relu_pool_kernel', 'linear_smallm_kernel']
)
# combinations the dispatch cannot produce, with the reason
UNREACHABLE = {
    'conv_tc2_kernel<32 or 128, F16, *, true>': 'xr_ok takes BN 64 only',
    'conv_tc2_kernel<*, TF32, true, *>': 'folding and x reuse need the split input, which is fp16 only',
    'conv_tcflat_kernel with K splits folded': 'fold_ok refuses the A-reuse kernel',
}


def test_coverage():
    """The kernels the cases above were seen to launch cover every reachable instantiation.  Needs the cases of this
    module to have run first (pytest runs a module's tests in file order)."""
    if len(ASSERTED) < len(CASES):
        pytest.skip('run with the rest of the module')
    got = set()
    for _, kernels in ASSERTED.values():
        got |= kernels
    missing = [k for k in REACHABLE if k not in got]
    print(f'\ncovered {len(REACHABLE) - len(missing)} of {len(REACHABLE)} reachable instantiations:')
    for k in REACHABLE:
        cases = [cid for cid, (_, ks) in ASSERTED.items() if k in ks]
        print(f'  {k:48s} {", ".join(cases[:4])}')
    for k, why in UNREACHABLE.items():
        print(f'  unreachable: {k}: {why}')
    assert not missing, missing
