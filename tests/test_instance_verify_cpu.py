"""Verification of the instance trackers (row f21) without a GPU: g6d_instances_verify_update_host (the code the kernel
runs) against the numpy restatement in instance_verify_oracle.py and against the association's own drop rule, bit for
bit; and the trackers' host logic: which steps verify, the counts under re-detection, reset, redetect, boxes and partial
steps, the sequences a lost verdict marks, the decode of the verification rows, graph names and argument errors."""
import numpy as np
import pytest
import torch

import instance_verify_oracle as oracle
from gen6d_b200 import _lib
from gen6d_b200 import boxes as B
from gen6d_b200 import verify as V
from gen6d_b200.frames import FramePlan
from gen6d_b200.instance_track import (InstanceTracker, ObjectInstanceTracker, Schedule, host_associate, host_verify_update,
                                       mixed_name)
from gen6d_b200.track import PartialStep
from tests.test_instance_track_cpu import make_problem

DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def built():
    from gen6d_b200.build import build
    build()


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def random_slots(rng, n, max_misses, live_p):
    live = (rng.rand(n) < live_p).astype(np.int32)
    ids = np.where(live, rng.permutation(max(1000, n))[:n], -1).astype(np.int64)
    misses = np.where(live, rng.randint(0, max_misses + 1, n), 0).astype(np.int32)
    return live, ids, misses


def run_twin(lost, verified, max_misses, live, ids, misses):
    live, ids, misses = live.copy(), ids.copy(), misses.copy()
    dropped = host_verify_update(lost, verified, max_misses, live, ids, misses)
    return live, ids, misses, dropped


# ------------------------------------------------------------------------------------------ the update rule
@pytest.mark.parametrize('M', [1, 2, 4])
@pytest.mark.parametrize('K', [1, 3])
@pytest.mark.parametrize('S', [1, 5])
@pytest.mark.parametrize('max_misses', range(4))
def test_host_twin_equals_oracle(M, K, S, max_misses):
    rng = np.random.RandomState(1000 * M + 100 * K + 10 * S + max_misses)
    n = M * K * S
    for trial in range(60):
        live, ids, misses = random_slots(rng, n, max_misses, rng.choice([0.0, 0.5, 1.0]))
        mode = trial % 5
        lost = np.ones(n, np.int32) if mode == 0 else np.zeros(n, np.int32) if mode == 1 else (rng.rand(n) < 0.5).astype(np.int32)
        seq_verified = rng.rand(S) < (1.0 if mode < 3 else 0.6)        # unverified rows: whole sequences, as a step masks them
        verified = np.tile(seq_verified, M * K).astype(np.int32)
        if mode == 4:
            verified = np.zeros(n, np.int32)
        got = run_twin(lost, verified, max_misses, live, ids, misses)
        want = oracle.verify_update(lost, verified, max_misses, live, ids, misses)
        for g, w, k in zip(got, want, ('live', 'ids', 'misses', 'dropped')):
            assert same(g, w), (trial, k, g, w)
        skip = (verified == 0) | (live == 0)
        assert same(got[0][skip], live[skip]) and same(got[1][skip], ids[skip]) and same(got[2][skip], misses[skip])


def test_drop_equals_the_association_drop():
    """A verification where every row is judged lost drops exactly what a re-detection with no detection drops."""
    rng = np.random.RandomState(7)
    for trial in range(200):
        p = make_problem(rng)
        n = len(p['live'])
        live, ids, misses = p['live'].copy(), p['ids'].copy(), p['misses'].copy()
        *_, dropped = host_associate(p['det'], np.zeros(n, np.int32), p['init'], p['cams'], p['center'], p['res'], p['gate'],
                                     p['max_misses'], p['F'], p['r'], p['prev'], live, ids, misses, p['next_id'].copy(),
                                     p['park'].copy(), p['ring'].copy(), p['count'].copy())
        got = run_twin(np.ones(n, np.int32), np.ones(n, np.int32), p['max_misses'], p['live'], p['ids'], p['misses'])
        for g, w, k in zip(got, (live, ids, misses, dropped), ('live', 'ids', 'misses', 'dropped')):
            assert same(g, w), (trial, k)


def test_update_arguments_are_checked():
    z = np.zeros(2, np.int32)
    with pytest.raises(_lib.Gen6DLibraryError, match='max_misses'):
        host_verify_update(z, z, -1, z.copy(), np.zeros(2, np.int64), z.copy())
    with pytest.raises(ValueError, match='contiguous'):
        host_verify_update(z, z, 0, z.astype(np.int64), np.zeros(2, np.int64), z.copy())


def test_entry_points_are_declared_and_bound():
    names = {'g6d_instances_verify_update', 'g6d_instances_verify_update_host'}
    assert names <= set(_lib.header_symbols())
    assert names <= set(_lib._SIGNATURES)


# ------------------------------------------------------------------------------------------ the tracker's host logic
class _FakeTracker(InstanceTracker):
    """An InstanceTracker's host planning without a GPU: _run plans and counts verification as the real one does, and
    returns results whose slots are all live; the sequences in `lose` are judged lost on every verifying step."""

    def __init__(self, S, schedule, E=None, every=None, lost_score=None, M=2, K=1):
        class Est:
            detector = type('D', (), {'device': DEV})()
            cfg = {'ref_resolution': 128}

            def _generation(self):
                return 0
        self.est, self._gen, self.S, self.M, self.K, self.schedule = Est(), 0, S, M, K, schedule
        self.redetect_every = E
        self._pending, self._since = True, 0
        self._schedule = Schedule(S, E, schedule == 'staggered')
        self._verify = V.Schedule(every, lost_score)
        self._vsince = np.zeros(S, np.int64)
        self._drawer, self.runs, self.lose = None, [], set()
        n = M * K * S
        self._state = {'live': torch.zeros(n, dtype=torch.int32), 'ids': torch.full((n,), -1, dtype=torch.int64),
                       'misses': torch.zeros(n, dtype=torch.int32), 'ring': torch.zeros(n, 1, 8, 2), 'count': torch.zeros(n, dtype=torch.int32)}

    def _run(self, frames, Ks, out, kind, part=None, det_seq=None, boxes=None):
        S, stepped, refining, check = self._verify_plan(kind, part, det_seq)
        self.runs.append((kind, check, stepped.copy(), refining[:len(stepped)].copy()))
        res = []
        for _ in range(self.K):
            inter = {}
            if check:
                lost = np.zeros((S, self.M), bool)
                lost[:len(stepped)] = np.isin(stepped, list(self.lose))[:, None] & refining[:len(stepped), None]
                inter['verify'] = {'lost': lost}
            res.append((np.zeros(S), np.zeros(S), np.zeros((S, self.M), np.int64), inter))
        self._verify_done(stepped, refining, check)
        return res


def _frames(n):
    return [np.zeros((8, 8, 3), np.uint8)] * n, [np.eye(3)] * n


def reference(S, every, steps):
    """Which steps verify, restated: steps lists per step (stepped sequences, re-detecting ones); a step verifies when a
    stepped sequence that does not re-detect has taken `every` steps since its last re-detection or verification."""
    since, out = np.zeros(S, np.int64), []
    for t, (stepped, det) in enumerate(steps):
        refining = [s for s in stepped if s not in det]
        v = any(since[s] + 1 >= every for s in refining)
        for s in stepped:
            since[s] = 0 if (s in det or v) else since[s] + 1
        if v:
            out.append(t)
    return out


def drive(trk, T):
    for _ in range(T):
        trk.step(*_frames(trk.S))
    return [t for t, r in enumerate(trk.runs) if r[1]]


@pytest.mark.parametrize('every', range(1, 7))
def test_which_steps_verify_lockstep(every):
    for E in (None, 1, 3, 7):
        trk = _FakeTracker(3, 'lockstep', E, every)
        got = drive(trk, 30)
        det = [t for t, r in enumerate(trk.runs) if r[0] == 'detect']
        want = [t for t in range(30) if t not in det and (t - max(d for d in det if d <= t)) % every == 0]
        assert got == want, (E, got, want)


@pytest.mark.parametrize('every', range(1, 7))
@pytest.mark.parametrize('schedule', ['per_sequence', 'staggered'])
def test_which_steps_verify_per_sequence(every, schedule):
    for S in range(1, 13):
        for E in ((None,) if schedule == 'per_sequence' else ()) + (1, 2, 5, 12):
            trk = _FakeTracker(S, schedule, E, every)
            got = drive(trk, 25)
            steps = [(list(r[2]), set(np.asarray(r[2])[~r[3]].tolist())) for r in trk.runs]
            assert got == reference(S, every, steps), (S, E)
            if schedule == 'staggered' and E > 1 and S >= E:
                kinds = [r[0] for r in trk.runs]
                assert set(kinds[1:]) == {'mixed'}                       # every step after the first is mixed ...
                # ... and still some verify, whenever a sequence refines verify_every steps between its re-detections
                assert bool(got) == (every < E), (S, E, every)
                # the re-detecting rows of a verifying step are not verified
                for t in got:
                    assert trk.runs[t][3].any() and not trk.runs[t][3].all()


def test_counts_under_reset_redetect_boxes_and_partial_steps():
    S, box = 4, np.array([[0, 0, 4, 4, 1]], np.float32)
    trk = _FakeTracker(S, 'per_sequence', None, 3)
    trk.step(*_frames(S))                                               # detect: every count restarts
    trk.step(*_frames(S))
    assert trk._vsince.tolist() == [1, 1, 1, 1]
    trk.reset([1])
    trk.redetect([2])
    assert trk._vsince.tolist() == [1, 0, 0, 1]
    trk.step(*_frames(S))                                               # mixed: 1 and 2 re-detect, 0 and 3 count
    assert not trk.runs[-1][1] and trk._vsince.tolist() == [2, 0, 0, 2]
    trk.step(*_frames(2), sequences=[3, 1])                             # partial: 3 reaches 3 and 1 is verified with it
    kind, check, stepped, refining = trk.runs[-1]
    assert check and stepped.tolist() == [1, 3] and refining.all()
    assert trk._vsince.tolist() == [2, 0, 0, 0]
    trk.step(*_frames(S), boxes=[box, None, None, None])                # 0 re-detects from boxes: not verified, restarts
    kind, check, stepped, refining = trk.runs[-1]
    assert kind == 'mixed' and not check and refining.tolist() == [False, True, True, True]
    assert trk._vsince.tolist() == [0, 1, 1, 1]
    trk.step(*_frames(S), boxes=[None, box, None, None])
    trk.step(*_frames(S))                                               # 2 and 3 reach 3: 0, 2, 3 verified
    kind, check, stepped, refining = trk.runs[-1]
    assert check and kind == 'refine' and trk._vsince.tolist() == [0, 0, 0, 0]
    # lockstep: a step with boxes re-detects every sequence and never verifies
    lock = _FakeTracker(2, 'lockstep', None, 1)
    lock.step(*_frames(2))
    lock.step(*_frames(2), boxes=[box, box])
    assert [r[1] for r in lock.runs] == [False, False]
    lock.step(*_frames(2))
    assert lock.runs[-1][1]
    lock.reset()
    assert lock._vsince.tolist() == [0, 0]


@pytest.mark.parametrize('schedule', ['lockstep', 'per_sequence', 'staggered'])
def test_lost_sequences_become_due(schedule):
    S = 5
    trk = _FakeTracker(S, schedule, 100 if schedule == 'staggered' else None, 2, lost_score=0.5)
    trk.lose = {1, 3}
    trk.step(*_frames(S))
    trk.step(*_frames(S))
    assert not trk.detecting().any()
    trk.step(*_frames(S))                                               # verifies, judges 1 and 3 lost
    assert trk.runs[-1][1]
    want = np.full(S, True) if schedule == 'lockstep' else np.isin(np.arange(S), [1, 3])
    np.testing.assert_array_equal(trk.detecting(), want)
    trk.lose = set()
    trk.step(*_frames(S))                                               # they re-detect
    assert trk.runs[-1][0] == ('detect' if schedule == 'lockstep' else 'mixed')
    assert not trk.detecting().any()
    if schedule != 'lockstep':                                          # a due sequence given None stays due
        trk.lose = {0}
        trk.step(*_frames(S))                                           # 0, 2 and 4 reach 2: verified, 0 lost
        assert trk.runs[-1][1] and trk.detecting().tolist() == [True, False, False, False, False]
        trk.step(*_frames(S), boxes=[None] * S)
        assert trk.detecting()[0]
    # partial steps mark only listed sequences
    part = _FakeTracker(S, 'per_sequence', None, 1, lost_score=0.5)
    part.step(*_frames(S))
    part.lose = {0, 4}
    part.step(*_frames(2), sequences=[4, 2])
    assert part.detecting().tolist() == [False, False, False, False, True]
    # thresholds None: verify and report, never mark
    quiet = _FakeTracker(S, schedule, 100 if schedule == 'staggered' else None, 1)
    quiet.lose = set(range(S))
    drive(quiet, 3)
    assert quiet.runs[-1][1] and not quiet.detecting().any()


def test_object_set_marks_a_sequence_lost_by_any_object():
    S = 3
    trk = _FakeTracker(S, 'per_sequence', None, 1, lost_score=0.0, K=2)

    def run(frames, Ks, out, kind, part=None, det_seq=None, boxes=None):
        S_, stepped, refining, check = trk._verify_plan(kind, part, det_seq)
        res = [(None, None, np.zeros((S_, 2), np.int64), {'verify': {'lost': np.zeros((S_, 2), bool)}} if check else {})
               for _ in range(2)]
        if check:
            res[1][3]['verify']['lost'][2, 1] = True                    # object 1, sequence 2, slot 1
        trk._verify_done(stepped, refining, check)
        return res
    trk._run = run
    trk.step(*_frames(S))
    trk.step(*_frames(S))
    assert trk.detecting().tolist() == [False, False, True]


def test_verification_rows_decode():
    """_verify_results: the rows of object o in [S, M] order, empty slots and non-refining rows masked, 'dropped' per
    object ascending."""
    M, K, S = 2, 3, 4
    n = M * K * S
    trk = _FakeTracker(S, 'per_sequence', None, 1, lost_score=0.5, M=M, K=K)
    rng = np.random.RandomState(3)
    vals = rng.rand(n, 10)
    vals[:, 5] = rng.rand(n) < 0.5
    checked = V.decode(vals, n)
    dropped = np.where(rng.rand(n) < 0.3, rng.permutation(n) + 100, -1).astype(np.int64)
    refining = np.array([True, False, True, True])
    ids = [np.where(rng.rand(S, M) < 0.7, 1, -1).astype(np.int64) for _ in range(K)]
    res = [(None, None, ids[o], {}) for o in range(K)]
    trk._verify_results(res, checked, dropped, refining, S)
    for o in range(K):
        v = res[o][3]['verify']
        for s in range(S):
            for m in range(M):
                row = (m * K + o) * S + s
                keep = ids[o][s, m] >= 0 and refining[s]
                assert v['lost'][s, m] == (keep and bool(vals[row, 5]))
                assert (v['score'][s, m] == np.float32(vals[row, 3])) if keep else np.isnan(v['score'][s, m])
                assert keep or np.isnan(v['window_center'][s, m]).all()
        rows = [(m * K + o) * S + s for m in range(M) for s in range(S)]
        assert v['dropped'] == sorted(int(dropped[r]) for r in rows if dropped[r] >= 0)
        assert set(v) == set(checked) | {'dropped'}


def test_graph_names_are_apart():
    part = PartialStep(8, 2, [0, 3, 5], np.zeros(8, bool), np.ones(8, bool), 1)
    plan = FramePlan([(48, 64), (40, 56)])
    wraps = [lambda n: n, part.name, lambda n: (n, 'draw', ('raw',)), plan.key, plan.device_key,
             lambda n: plan.key(part.name(n)), lambda n: B.graph_name(n, 4), lambda n: part.name(B.graph_name(n, 8))]
    bases = ['refine', 'detect', mixed_name(8, 2), mixed_name(4, 4), mixed_name(8, (2, 2))]
    keys = [(None, None), (0.5, None), (None, 0.25), (np.inf, 1.0)]
    f20 = {V.graph_name(b, k) for b in ('track_refine0', 'track_refine1') for k in keys}
    existing = {w(b) for w in wraps for b in bases + ['track_refine0', 'track_refine1', 'verify_poses'] + list(f20)}
    verifying = {w(V.graph_name(b, k)) for w in wraps for b in ('refine', mixed_name(8, 2), mixed_name(4, 4), mixed_name(8, (2, 2)))
                 for k in keys}
    assert len(verifying) == len(wraps) * 4 * len(keys)
    assert not verifying & existing


def test_argument_errors():
    for bad in (0, -1, 1.5, 'x', True):
        with pytest.raises(ValueError, match='verify_every'):
            ObjectInstanceTracker(None, 2, verify_every=bad)
    with pytest.raises(ValueError, match='verify_every too'):
        ObjectInstanceTracker(None, 2, lost_score=0.0)
    with pytest.raises(ValueError, match='verify_every too'):
        ObjectInstanceTracker(None, 2, lost_gate=0.5)
    with pytest.raises(ValueError, match='NaN'):
        ObjectInstanceTracker(None, 2, verify_every=1, lost_score=float('nan'))
    with pytest.raises(ValueError, match='lost_gate'):
        ObjectInstanceTracker(None, 2, verify_every=1, lost_gate=-1.0)


def test_no_verification_without_verify_every():
    trk = _FakeTracker(3, 'per_sequence', 2, None)
    assert not any(r[1] for r in trk.runs) and not drive(trk, 12)
    assert InstanceTracker._verify.every is None
