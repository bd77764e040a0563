"""Partial tracker steps (row f17) without a GPU: the host plan of a step over a subset of the sequences (bucket,
padding, step kind, gather and scatter rows, graph names), the compact graph body's gather and scatter on CPU tensors,
and the argument errors, raised before anything is enqueued."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gen6d_b200 import draw as dr
from gen6d_b200 import frames as fr
from gen6d_b200.track import PartialStep, Tracker, _bucket, _compact_fn, _step_kind


def _lists(S, rng):
    """Ascending and permuted lists of every length 1..S."""
    out = []
    for a in range(1, S + 1):
        pick = np.sort(rng.choice(S, a, replace=False))
        out += [pick.tolist(), rng.permutation(pick).tolist()]
    return out


@pytest.mark.parametrize('S', [1, 3, 4, 10])
def test_bucket_and_padding(S):
    rng = np.random.RandomState(S)
    pending, f32 = np.zeros(S, bool), np.ones(S, bool)
    for seqs in _lists(S, rng):
        p = PartialStep(S, 1, seqs, pending, f32, 1)
        a = len(seqs)
        assert p.a == a and p.lockstep == (a == S)
        assert p.b == (S if a == S else _bucket(a, S)) and a <= p.b <= S and (p.b & (p.b - 1) == 0 or p.b == S)
        # the listed sequences ascending, then the last of them repeated
        assert p.seq.tolist() == sorted(seqs) + [max(seqs)] * (p.b - a)
        assert p.sequences.tolist() == seqs and p.sequences.dtype == np.int64
        # pos maps the caller's entries to their compact rows, order the compact rows to the caller's entries
        assert [p.seq[p.pos[i]] for i in range(a)] == seqs
        assert [seqs[i] for i in p.order] == p.seq.tolist()
        assert p.compact(list(range(a))) == p.order.tolist()


@pytest.mark.parametrize('K', [1, 3])
@pytest.mark.parametrize('S', [1, 3, 4, 10])
def test_gather_and_scatter_rows(S, K):
    rng = np.random.RandomState(10 * S + K)
    pending, f32 = np.zeros(S, bool), np.ones(S, bool)
    for seqs in _lists(S, rng):
        p = PartialStep(S, K, seqs, pending, f32, 1)
        a, b, n = p.a, p.b, K * S
        g, s = p.gather.reshape(K, b), p.scatter.reshape(K, b)
        assert p.gather.dtype == p.scatter.dtype == np.int64
        for o in range(K):
            assert (g[o] == o * S + p.seq).all()                             # object-major tracker rows
            assert (s[o, :a] == o * S + p.seq[:a]).all()                     # real rows go home
            assert (s[o, a:] == n + o * b + np.arange(a, b)).all()           # padding rows to their own scratch copy
        assert len(set(p.scatter.tolist())) == K * b                          # every target once: no row written twice
        assert set(p.scatter[p.scatter < n].tolist()) == {o * S + q for o in range(K) for q in seqs}


def test_step_kind_from_listed_flags_only():
    S = 6
    pending = np.array([1, 1, 0, 0, 0, 0], bool)
    f32 = np.array([1, 1, 1, 1, 0, 0], bool)
    cases = {(0,): 'full', (1, 0): 'full', (2,): 'refine', (3, 2): 'refine', (4, 5): 'refine', (5,): 'refine',
             (0, 2): 'mixed', (3, 4): 'mixed', (1, 5, 2): 'mixed', tuple(range(S)): 'mixed'}
    for seqs, kind in cases.items():
        p = PartialStep(S, 1, list(seqs), pending, f32, 1)
        assert p.kind == kind == _step_kind(pending[list(seqs)], f32[list(seqs)], 1), seqs
        assert p.pending.tolist() == pending[p.seq].tolist() and p.f32.tolist() == f32[p.seq].tolist()
    # the tracker-wide flags would make each of these a mixed step
    assert _step_kind(pending, f32, 1) == 'mixed'
    with pytest.raises(ValueError, match='refine_iter'):
        PartialStep(S, 1, [0, 2], pending, f32, 0)
    assert PartialStep(S, 1, [2, 3], pending, f32, 0).kind == 'refine'


def test_plan_flags_are_copies():
    pending, f32 = np.ones(4, bool), np.ones(4, bool)
    p = PartialStep(4, 1, [1, 2], pending, f32, 1)
    pending[:], f32[:] = False, False
    assert p.pending.all() and p.f32.all() and p.kind == 'full'


def _lockstep_bases(S):
    bases = ['track_full', 'track_refine0', 'track_refine1'] + [f'track_mixed{b}' for b in range(S + 1)]
    plan = fr.FramePlan([(48, 64), (32, 40)] * 2)
    bases += [(plan.key('track_mixed'), (b, c)) for b in range(3) for c in range(3)]
    return bases


def _names(base):
    """Every name a step graph of `base` can take: with and without drawing, numpy / mixed-size / device keys."""
    plan = fr.FramePlan([(48, 64), (32, 40)])
    draws = [lambda n: n] + [lambda n, k=k: dr.StepDrawer.name(SimpleNamespace(kinds=k), n)
                             for k in (('raw',), ('smoothed',), ('raw', 'smoothed'))]
    keys = [lambda n: n, plan.key, plan.device_key, lambda n: plan.device_key(n, True)]
    return {key(d(base)) for d in draws for key in keys}


@pytest.mark.parametrize('S', [3, 4, 10])
def test_graph_names_are_apart_from_lockstep_names(S):
    lock = set().union(*(_names(b) for b in _lockstep_bases(S)))
    pending, f32 = np.zeros(S, bool), np.ones(S, bool)
    part, per_b = set(), {}
    for a in range(1, S):
        p = PartialStep(S, 1, list(range(a)), pending, f32, 1)
        for base in _lockstep_bases(S):
            names = _names(p.name(base))
            part |= names
            per_b.setdefault(p.b, set()).update(names)
    assert not part & lock
    bs = sorted(per_b)
    assert all(not per_b[x] & per_b[y] for i, x in enumerate(bs) for y in bs[i + 1:])    # buckets apart too


def test_results_in_the_callers_order():
    S, seqs = 8, [6, 1, 4]
    pending, f32 = np.zeros(S, bool), np.ones(S, bool)
    p = PartialStep(S, 1, seqs, pending, f32, 1)
    b = p.b
    assert b == 4 and p.seq.tolist() == [1, 4, 6, 6]
    raw = np.arange(b, dtype=np.float32)[:, None, None] + np.zeros((b, 3, 4), np.float32)
    inter = {'refine_poses': [raw.astype(np.float64), raw], 'bbox_pts': np.arange(b)[:, None, None] + np.zeros((b, 8, 2)),
             'drawn': {'raw': ['d1', 'd4', 'd6', 'pad']}}
    r, sm, got = p.results(raw, raw.astype(np.float64), inter)
    want = [p.seq.tolist().index(s) for s in seqs]
    assert r[:, 0, 0].tolist() == want and sm[:, 0, 0].tolist() == want
    assert [c[:, 0, 0].tolist() for c in got['refine_poses']] == [want, want]
    assert got['bbox_pts'][:, 0, 0].tolist() == want and got['drawn'] == {'raw': ['d6', 'd1', 'd4']}
    assert got['sequences'].tolist() == seqs
    # a mixed step: compact rows 1 and 3 (sequence 4 and the padding copy of 6) and 2 (sequence 6) re-initialised
    mixed = {'reinit': np.array([1, 2, 3]), 'sel_ref_idx': np.array([10, 20, 30]), 'det_que_img': [b'x', b'y', b'z'],
             'refine_poses': [raw], 'smoothed_pts': np.zeros((b, 8, 2))}
    _, _, got = p.results(raw, raw, mixed)
    assert got['reinit'].tolist() == [4, 6] and got['sel_ref_idx'].tolist() == [10, 20] and got['det_que_img'] == [b'x', b'y']
    assert got['smoothed_pts'].shape == (3, 8, 2)


@pytest.mark.parametrize('K', [1, 2])
def test_compact_body_writes_only_the_listed_rows(K):
    """_compact_fn with a stand-in step body on CPU tensors: the body sees the gathered rows in compact order, the listed
    rows get its results, every other row keeps its bytes, and a padding row's result reaches no row."""
    S, num, seqs = 5, 3, [3, 0, 4]
    p = PartialStep(S, K, seqs, np.zeros(S, bool), np.ones(S, bool), 1)
    b = p.b
    prev = torch.arange(K * S * 12, dtype=torch.float64).reshape(K * S, 12)
    ring = torch.randn(K * S, num, 8, 2)
    count = torch.arange(K * S, dtype=torch.int32)
    seen = {}

    def body(frames, cams, prev_c, ring_c, count_c, *rest):
        seen.update(prev=prev_c.clone(), rest=rest)
        poses = prev_c + 1000
        poses.view(K, b, 12)[:, p.a:] = -1                     # padding rows: a canary that must land nowhere
        ring_c.add_(1)
        count_c.add_(1)
        return torch.zeros(4, dtype=torch.uint8), poses, ring_c, count_c

    g = _compact_fn(body, False)
    gather, scatter = [torch.from_numpy(t) for t in (p.gather, p.scatter)]
    buf, p2, r2, c2 = g(None, None, prev, ring.clone(), count.clone(), gather, scatter, 'extra')
    assert seen['rest'] == ('extra',) and torch.equal(seen['prev'], prev[gather])
    rows = np.concatenate([o * S + np.asarray(sorted(seqs)) for o in range(K)])
    others = np.setdiff1d(np.arange(K * S), rows)
    assert torch.equal(p2[rows], prev[rows] + 1000) and torch.equal(p2[others], prev[others])
    assert torch.equal(r2[rows], ring[rows] + 1) and torch.equal(r2[others], ring[others])
    assert torch.equal(c2[rows], count[rows] + 1) and torch.equal(c2[others], count[others])
    assert p2.shape == prev.shape and r2.shape == ring.shape and c2.shape == count.shape and (p2 != -1).all()
    # a full step's body takes no previous poses; they pass through
    full = _compact_fn(lambda f, c, r, n: (None, torch.zeros(K * b, 12, dtype=torch.float64), r, n), True)
    _, p3, _, _ = full(None, None, prev, ring, count, gather, scatter)
    assert (p3[rows] == 0).all() and torch.equal(p3[others], prev[others])


# ------------------------------------------------------------------------------------------ errors
def _host_tracker(S=4, drawer=None):
    t = Tracker.__new__(Tracker)               # the state and argument checks only: no estimator, no GPU
    t.est = SimpleNamespace(cfg={'refine_iter': 1}, _generation=lambda: 0)
    t._gen, t.S, t.num, t._drawer = 0, S, 5, drawer
    t.reset()
    return t


BAD = {'duplicate': ([1, 1], 2), 'high': ([4], 1), 'negative': ([-1], 1), 'empty': ([], 0),
       'few_frames': ([0, 2], 1), 'many_frames': ([0], 2)}


@pytest.mark.parametrize('bad', sorted(BAD))
def test_bad_lists_are_rejected_before_anything_runs(bad):
    seqs, n = BAD[bad]
    t = _host_tracker()
    t.start(np.zeros((4, 3, 4), np.float32))
    t.reset([2])
    state = [a.copy() for a in (t._prev, t._ring, t._count, t._pending, t._f32)]
    frames = [np.zeros((8, 8, 3), np.uint8)] * n
    with pytest.raises(ValueError):
        t.step(frames, [np.eye(3)] * n, sequences=seqs)
    for x, y in zip(state, (t._prev, t._ring, t._count, t._pending, t._f32)):
        assert x.tobytes() == y.tobytes()


def test_length_mismatches_are_rejected():
    t = _host_tracker()
    f = [np.zeros((8, 8, 3), np.uint8)] * 2
    with pytest.raises(ValueError, match='Ks'):
        t.step(f, [np.eye(3)] * 3, sequences=[0, 1])
    with pytest.raises(ValueError, match='draw='):
        t.step(f, [np.eye(3)] * 2, out={'raw': [None, None]}, sequences=[0, 1])
    t._drawer = SimpleNamespace()
    with pytest.raises(ValueError, match='out'):
        t.step(f, [np.eye(3)] * 2, out={'raw': [None]}, sequences=[0, 1])
    with pytest.raises(ValueError, match='2 sequences'):
        PartialStep(4, 1, [0, 3], np.zeros(4, bool), np.ones(4, bool), 1).check(f, [np.eye(3)] * 2, {'raw': [1, 2, 3]})
