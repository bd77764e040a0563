"""Per-sequence re-detection of the instance trackers without a GPU: g6d_instances_associate_sequences_host (the code the
device kernel runs) against the lockstep association it generalises, the refine-only set-up and the numpy restatement in
instance_assoc_oracle.py, bit for bit; and the host planning of the per-sequence schedules (flags, counters, staggered
phases, graph keys, padding, errors)."""
import numpy as np
import pytest

from tests import instance_assoc_oracle as oracle
from tests.test_instance_track_cpu import OUTS, STATE, make_problem
from tests.test_objects_instance_track_cpu import G6D_EINVAL, make_set_problem

ARGS = ('det', 'valid', 'init', 'cams', 'centers', 'res', 'gate', 'max_misses', 'F', 'r', 'prev')


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200 import _lib
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def _copy(p):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}


def run_sequences(p, det_index, det_rows=None):
    """host_associate_sequences on a copy of problem p -> every output and state array.  det_rows: the problem's detection
    arrays already in the batch layout (default: p's own, the identity layout)."""
    from gen6d_b200.instance_track import host_associate_sequences
    q = _copy(p)
    if det_rows is not None:
        q.update(det_rows)
    outs = host_associate_sequences(np.asarray(det_index), *[q[k] for k in ARGS], *[q[k] for k in STATE])
    return {**dict(zip(OUTS, outs)), **{k: q[k] for k in STATE}}


def run_objects(p):
    from gen6d_b200.instance_track import host_associate_objects
    q = _copy(p)
    outs = host_associate_objects(*[q[k] for k in ARGS], *[q[k] for k in STATE])
    return {**dict(zip(OUTS, outs)), **{k: q[k] for k in STATE}}


def same(g, w):
    g, w = np.asarray(g), np.asarray(w)
    return g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g.view(np.uint8), w.view(np.uint8))


def assert_same(got, want, tag=''):
    for k in OUTS + STATE:
        assert same(got[k], want[k]), (tag, k, got[k], want[k])


def set_problem(rng, K, M, F, r, S=None):
    p, K_, S_, M_ = make_set_problem(rng, K, S=S or int(rng.randint(1, 6)), M=M, F=F, r=r)
    return p, K_, S_, M_


# ------------------------------------------------------------------------------------------ identity and all -1
FR = [(3, 1), (2, 2), (1, 3), (4, 2)]


@pytest.mark.parametrize('K', [1, 3])
@pytest.mark.parametrize('M', [1, 4])
@pytest.mark.parametrize('F,r', FR)
def test_identity_equals_the_lockstep_association(lib, K, M, F, r):
    """det_index the identity with D = S: every output and state array equals g6d_instances_associate_objects_host."""
    rng = np.random.RandomState(10 * K + M + 100 * F + 1000 * r)
    for trial in range(120):
        p, _, S, _ = set_problem(rng, K, M, F, r)
        assert_same(run_sequences(p, np.arange(S)), run_objects(p), trial)


def test_identity_equals_the_single_object_association(lib):
    from tests.test_instance_track_cpu import run_both
    rng = np.random.RandomState(21)
    for trial in range(300):
        p = make_problem(rng)
        if p['r'] < 1:
            continue
        want, _ = run_both(p)
        q = {**p, 'centers': np.asarray(p['center'], np.float64).reshape(1, 3)}
        assert_same(run_sequences(q, np.arange(len(p['cams']))), want, trial)


def refine_setup(p, K, S, M):
    """The set-up _refine_fn's graph does for every row, in the association's work / list layout."""
    G = M * K
    live, prev, park = p['live'], p['prev'], p['park']
    start = np.where((live != 0)[:, None], prev, park).reshape(G, S, 12)
    work = np.concatenate([start, start], 1).reshape(2 * G * S, 12)
    f = live.astype(np.uint8).reshape(G, S)
    flags0 = np.concatenate([f, f], 1).reshape(-1)
    real = (np.arange(G)[:, None] * 2 * S + np.arange(S)[None]).reshape(-1).astype(np.int32)
    return work, flags0, real


@pytest.mark.parametrize('K', [1, 3])
@pytest.mark.parametrize('F,r', FR[:3])
def test_no_detection_is_the_refine_setup(lib, K, F, r):
    """Every entry -1 (D = 0): the refine step's start poses and flags, r iterations over every real row, nothing else; no
    state byte changes."""
    rng = np.random.RandomState(7 + K + F)
    for trial in range(60):
        p, _, S, M = set_problem(rng, K, int(rng.choice([1, 2, 4])), F, r)
        empty = {'det': np.zeros((0, 4), np.float32), 'valid': np.zeros(0, np.int32), 'init': np.zeros((0, 12))}
        got = run_sequences(p, np.full(S, -1), empty)
        work, flags0, real = refine_setup(p, K, S, M)
        assert same(got['work'], work) and same(got['flags0'], flags0), trial
        assert same(got['lists'], np.tile(real, r)), trial
        assert (got['spawned'] == 0).all() and (got['dropped'] == -1).all() and (got['det_slot'] == -1).all()
        for k in STATE:
            assert same(got[k], p[k]), (trial, k)


# ------------------------------------------------------------------------------------------ random masks
def random_case(rng, K, F=None, r=None):
    """A set problem, a random detecting subset with a permuted det_index (D its bucket, padding rows filled with another
    sequence's detections) -> (p, det_index, batch detection arrays, K, S, M, D)."""
    p, K, S, M = set_problem(rng, K, int(rng.choice([1, 2, 3, 4])), rng.randint(1, 5) if F is None else F,
                             rng.randint(1, 4) if r is None else r, S=int(rng.randint(1, 9)))
    from gen6d_b200.track import _bucket
    det_seqs = np.flatnonzero(rng.rand(S) < rng.uniform(0, 1))
    m = len(det_seqs)
    D = _bucket(m, S) if rng.rand() < 0.7 else int(rng.randint(m, S + 1))
    det_index = np.full(S, -1)
    det_index[det_seqs] = rng.permutation(D)[:m]
    G = M * K
    batch = {'det': rng.randn(G * D, 4).astype(np.float32), 'valid': rng.randint(0, 2, G * D).astype(np.int32),
             'init': rng.randn(G * D, 12)}
    for s in det_seqs:                                    # the sequence's own detections go to its batch row
        for g in range(G):
            for k in ('det', 'valid', 'init'):
                batch[k][g * D + det_index[s]] = p[k][g * S + s]
    return p, det_index, batch, K, S, M, D


def subset_problem(p, K, S, M, seqs):
    """The problem restricted to sequences `seqs` (ascending), in the lockstep layout of len(seqs) sequences."""
    G, m = M * K, len(seqs)
    rows = np.asarray([g * S + s for g in range(G) for s in seqs], np.int64)
    q = _copy(p)
    for k in ('det', 'valid', 'init', 'prev', 'live', 'ids', 'misses', 'park', 'ring', 'count'):
        q[k] = np.ascontiguousarray(p[k][rows])
    q['cams'] = np.ascontiguousarray(p['cams'][seqs])
    return q, rows


@pytest.mark.parametrize('K', [1, 2])
def test_random_masks(lib, K):
    """Detecting pairs equal the oracle (K = 1) / the lockstep association (K = 2) on those sequences alone; the others
    get the refine set-up and keep their state; ids ascend over the detecting pairs; the lists follow the rule."""
    rng = np.random.RandomState(300 + K)
    n_spawn = n_mixed = 0
    for trial in range(400):
        p, det_index, batch, K_, S, M, D = random_case(rng, K)
        F, r, G = p['F'], p['r'], M * K
        got = run_sequences(p, det_index, batch)
        det_seqs = np.flatnonzero(det_index >= 0)
        others = np.flatnonzero(det_index < 0)
        m = len(det_seqs)
        n_mixed += 0 < m < S
        # the detecting sequences alone, through the lockstep association
        if m:
            q, rows = subset_problem(p, K, S, M, det_seqs)
            if K == 1:
                want = _copy(q)
                outs = oracle.associate(*[want[k] for k in ('det', 'valid', 'init', 'cams')], p['centers'][0], p['res'], p['gate'],
                                        p['max_misses'], F, r, want['prev'], *[want[k] for k in STATE])
                want.update(dict(zip(OUTS, outs)))
            else:
                want = run_objects(q)
            for k in ('live', 'ids', 'misses', 'park', 'ring', 'count', 'spawned', 'dropped', 'det_slot'):
                assert np.array_equal(np.asarray(got[k])[rows], np.asarray(want[k]).astype(got[k].dtype)), (trial, k)
            assert got['next_id'][0] == want['next_id'][0], trial
            n_spawn += int(np.asarray(want['spawned']).sum())
            # work rows and flags: subset row g*2m + x is full row g*2S + x (real) / g*2S + S + (x - m) (scratch), x over seqs
            wmap = np.asarray([g * 2 * S + (0 if x < m else S) + det_seqs[x % m] for g in range(G) for x in range(2 * m)])
            assert same(got['work'][wmap], np.asarray(want['work'], np.float64)), trial
            assert same(got['flags0'][wmap], np.asarray(want['flags0']).astype(np.uint8)), trial
            wl = np.asarray(want['lists']).reshape(max(F, r), G, m)
            for it in range(max(F, r)):
                for g in range(G):
                    for i, s in enumerate(det_seqs):
                        e = (it * G + g) * S + s if it < r else r * G * S + ((it - r) * G + g) * D + det_index[s]
                        assert got['lists'][e] == wmap[wl[it, g, i]], (trial, it, g, s)
        else:
            assert got['next_id'][0] == p['next_id'][0]
        # the non-detecting sequences: the refine set-up, their state untouched
        work, flags0, real = refine_setup(p, K, S, M)
        for s in others:
            st = np.arange(G) * S + s
            wr = np.concatenate([np.arange(G) * 2 * S + s, np.arange(G) * 2 * S + S + s])
            assert same(got['work'][wr], work[wr]) and same(got['flags0'][wr], flags0[wr]), (trial, s)
            for k in ('live', 'ids', 'misses', 'park', 'ring', 'count'):
                assert same(got[k][st], p[k][st]), (trial, s, k)
            assert (got['spawned'][st] == 0).all() and (got['dropped'][st] == -1).all() and (got['det_slot'][st] == -1).all()
            for it in range(r):
                assert np.array_equal(got['lists'][it * G * S + st], real[st]), (trial, s, it)
        # ids ascend over the detecting pairs in (object, sequence, slot) order
        spawned_ids = [got['ids'][(t * K + o) * S + s] for o in range(K) for s in range(S) for t in range(M)
                       if got['spawned'][(t * K + o) * S + s]]
        assert spawned_ids == list(range(p['next_id'][0], p['next_id'][0] + len(spawned_ids))), trial
        # the lists: r full iterations, then max(F-r, 0) over the D batch rows; padding rows use free scratch rows
        assert len(got['lists']) == r * G * S + max(F - r, 0) * G * D
        for it in range(max(F, r)):
            L = got['lists'][it * G * S:(it + 1) * G * S] if it < r else \
                got['lists'][r * G * S + (it - r) * G * D:r * G * S + (it - r + 1) * G * D]
            assert len(np.unique(L)) == len(L), (trial, it)                 # no row twice in one refiner stage
        unused = [j for j in range(D) if j not in set(det_index[det_seqs].tolist())]
        for k, j in enumerate(unused):
            for it in range(r, F):
                for g in range(G):
                    assert got['lists'][r * G * S + ((it - r) * G + g) * D + j] == g * 2 * S + S + others[k], (trial, j)
    assert n_mixed > 100 and n_spawn > 100, (n_mixed, n_spawn)


def test_padding_detections_reach_no_row(lib):
    """The batch's padding rows are never read: changing them changes no output."""
    rng = np.random.RandomState(11)
    hit = 0
    for trial in range(200):
        p, det_index, batch, K, S, M, D = random_case(rng, 2, F=3, r=1)
        used = set(det_index[det_index >= 0].tolist())
        pad = [j for j in range(D) if j not in used]
        if not pad:
            continue
        hit += 1
        other = {k: v.copy() for k, v in batch.items()}
        for g in range(M * K):
            for j in pad:
                other['det'][g * D + j] = rng.randn(4) * 100
                other['valid'][g * D + j] = 1
                other['init'][g * D + j] = rng.randn(12)
        assert_same(run_sequences(p, det_index, other), run_sequences(p, det_index, batch), trial)
    assert hit > 30


@pytest.mark.parametrize('det_index,D,msg', [([0, 0], 2, 'both 0'), ([0, 2], 2, 'outside'), ([-2, 0], 1, 'outside'),
                                             ([0, 1], 3, '0 <= D <= S'), ([0, -1], -1, 'outside')])
def test_bad_det_index_is_rejected(lib, det_index, D, msg):
    from gen6d_b200 import _lib
    from gen6d_b200.instance_track import check_det_index, host_associate_sequences
    p, K, S, M = make_set_problem(np.random.RandomState(2), 1, S=2, M=2, F=2, r=1)
    Dp = max(D, 0)
    batch = {'det': np.zeros((M * K * Dp, 4), np.float32), 'valid': np.zeros(M * K * Dp, np.int32), 'init': np.zeros((M * K * Dp, 12))}
    q = {**_copy(p), **batch}
    live = q['live'].copy()
    with pytest.raises(_lib.Gen6DLibraryError, match=msg):
        host_associate_sequences(np.asarray(det_index), *[q[k] for k in ARGS], *[q[k] for k in STATE])
    np.testing.assert_array_equal(q['live'], live)
    with pytest.raises(ValueError):
        check_det_index(np.asarray(det_index), S, D)


def test_bad_arguments_are_rejected_before_any_launch(lib):
    """The device entry checks what it can without reading device memory: D within [0, S] and the pointers."""
    p, K, S, M = make_set_problem(np.random.RandomState(3), 1, S=2, M=2, F=1, r=1)
    before = lib.g6d_launch_count()
    args = [S, K, M, 1, 1, 3, None] + [None] * 5 + [1.0, 0.5, 1] + [None] * 8 + [3] + [None] * 6 + [None]
    assert lib.g6d_instances_associate_sequences(*args) == G6D_EINVAL
    assert b'g6d_instances_associate_sequences:' in lib.g6d_last_error()
    args[6] = p['valid'].ctypes.data                  # a det_index pointer, D still beyond S
    args[11] = p['centers'].ctypes.data
    assert lib.g6d_instances_associate_sequences(*args) == G6D_EINVAL
    assert b'0 <= D <= S' in lib.g6d_last_error()
    assert lib.g6d_launch_count() == before


def test_entry_points_are_declared_and_bound():
    from gen6d_b200 import _lib
    for n in ('g6d_instances_associate_sequences', 'g6d_instances_associate_sequences_host'):
        assert n in _lib.header_symbols() and n in _lib._SIGNATURES, n


# ------------------------------------------------------------------------------------------ planning
@pytest.mark.parametrize('S', range(1, 13))
def test_staggered_schedule_bounds_redetections(S):
    """The tracker's own Schedule stepped in lockstep: the first step detects every sequence, every later one at most
    ceil(S/E), and each sequence every E steps."""
    from gen6d_b200.instance_track import Schedule
    for E in range(1, 13):
        sch = Schedule(S, E, staggered=True)
        seqs = np.arange(S)
        last = np.full(S, -1)
        for step in range(3 * E + 2):
            det, kind = sch.plan(seqs, S)
            if step == 0:
                assert det.all() and kind == 'detect'
            else:
                assert det.sum() <= -(-S // E), (S, E, step, det)
                assert kind == ('refine' if not det.any() else 'detect' if det.all() else 'mixed')
                gaps = step - last[det]
                assert (last[det] == 0).all() or (gaps[last[det] > 0] == E).all(), (S, E, step)
            last[det] = step
            sch.advance(seqs)


def test_per_sequence_schedule_flags_and_counters():
    """Own flags and counters: marked sequences detect on their next step only, the periodic ones every E of their own
    steps, idle sequences keep their counters; padding rows never detect."""
    from gen6d_b200.instance_track import Schedule
    sch = Schedule(4, 3, staggered=False)
    assert sch.due().all()
    det, kind = sch.plan(np.array([1, 3, 3]), 2)                 # a partial step of 1 and 3, padded by 3
    assert det.tolist() == [True, True, False] and kind == 'mixed'
    sch.advance(np.array([1, 3]))
    assert sch.pending.tolist() == [True, False, True, False] and sch.count.tolist() == [0, 1, 0, 1]
    for _ in range(2):
        det, kind = sch.plan(np.array([1]), 1)
        assert not det.any() and kind == 'refine'
        sch.advance(np.array([1]))
    assert sch.count.tolist() == [0, 3, 0, 1]
    det, kind = sch.plan(np.arange(4), 4)
    assert det.tolist() == [True, True, True, False] and kind == 'mixed'
    sch.advance(np.arange(4))
    assert sch.count.tolist() == [1, 1, 1, 2] and not sch.pending.any()
    sch.pending[2] = True                                         # redetect([2])
    assert sch.plan(np.arange(4), 4)[0].tolist() == [False, False, True, False]
    none = Schedule(2, None, staggered=False)
    none.advance(np.arange(2))
    for _ in range(50):
        assert not none.due().any()
        none.advance(np.arange(2))


def test_staggered_restart_at_phase():
    from gen6d_b200.instance_track import Schedule, staggered_phases
    assert staggered_phases(10, 10).tolist() == list(range(10))
    assert staggered_phases(4, 3).tolist() == [0, 0, 1, 2]
    sch = Schedule(4, 3, staggered=True)
    sch.advance(np.arange(4))                                     # the first (marked) detection
    assert sch.count.tolist() == [1, 1, 2, 3]
    assert sch.plan(np.arange(4), 4)[0].tolist() == [False, False, False, True]
    sch.advance(np.arange(4))                                     # sequence 3's periodic detection restarts at 1
    assert sch.count.tolist() == [2, 2, 3, 1]
    sch.pending[0] = True                                         # reset([0]): back on its phase after the detection
    sch.advance(np.arange(4))
    assert sch.count.tolist() == [1, 3, 1, 2]


def test_mixed_plan_and_names():
    """plan_mixed: the re-detecting sequences gathered ascending, padded by repeating the last, their rows in det_index;
    per-size blocks for frames of two sizes; the (b, d) names apart from every lockstep and partial name."""
    from gen6d_b200 import frames as fr
    from gen6d_b200.instance_track import mixed_name, plan_mixed
    from gen6d_b200.track import PartialStep
    seq, blocks, det_index, d, key = plan_mixed(np.array([False, True, False, True, True, False]), None)
    assert seq.tolist() == [1, 3, 4, 4] and blocks is None and d == key == 4
    assert det_index.tolist() == [-1, 0, -1, 1, 2, -1]
    plan = fr.FramePlan(((480, 640), (400, 560), (480, 640), (400, 560)))
    seq, blocks, det_index, d, key = plan_mixed(np.array([True, True, True, False]), plan)
    assert blocks == [2, 1] and key == (2, 1) and d == 3
    assert sorted(seq.tolist()) == [0, 1, 2] and (seq[det_index[:3]] == [0, 1, 2]).all() and det_index[3] == -1
    names = {'detect', 'refine'}
    for b in range(1, 7):
        for dd in range(1, b):
            assert mixed_name(b, dd) not in names
            names.add(mixed_name(b, dd))
    part = PartialStep(6, 2, [4, 1], np.zeros(6, bool), np.ones(6, bool), 1)
    for base in list(names):
        assert part.name(base) not in names
    with pytest.raises(ValueError, match='twice'):
        PartialStep(6, 2, [1, 1], np.zeros(6, bool), np.ones(6, bool), 1)
    with pytest.raises(ValueError, match='outside'):
        PartialStep(6, 2, [6], np.zeros(6, bool), np.ones(6, bool), 1)


def test_schedule_arguments():
    from gen6d_b200.instance_track import SCHEDULES, check_args
    args = dict(num_sequences=2, max_instances=2, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1, min_score=None,
                nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5)
    for sch in ('lockstep', 'per_sequence'):
        check_args(**args, schedule=sch)
    check_args(**{**args, 'redetect_every': 3}, schedule='staggered')
    with pytest.raises(ValueError, match='redetect_every'):
        check_args(**args, schedule='staggered')
    with pytest.raises(ValueError, match='schedule'):
        check_args(**args, schedule='sometimes')
    assert SCHEDULES == ('lockstep', 'per_sequence', 'staggered')


def test_spread_fills_non_detecting_rows():
    from gen6d_b200.instance_track import _spread
    L, D = 2, 2
    a = np.arange(L * D * 3, dtype=np.float64).reshape(L * D, 3)
    got = _spread(a, L, D, np.array([1, -1, 0]), np.nan).reshape(L, 3, 3)
    np.testing.assert_array_equal(got[:, 0], a.reshape(L, D, 3)[:, 1])
    np.testing.assert_array_equal(got[:, 2], a.reshape(L, D, 3)[:, 0])
    assert np.isnan(got[:, 1]).all()
