"""The row-indexed refinement glue (g6d_glue_refine_problems_rows, g6d_glue_apply_refinements_rows) through their *_host
twins, without a GPU: every listed row must be bit-identical to that row of the object-indexed entry point called with
that row's dtype flag, only the listed rows may be written, and bad arguments must be rejected before any launch."""
import ctypes as C

import numpy as np
import pytest

from gen6d_b200 import _lib, glue

from test_track_objects_cpu import BUF, G6D_EINVAL, _random_poses, _sources, _views

SEEDS = (7, 8, 11)


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


@pytest.fixture(scope='module')
def dbs():
    from gen6d_b200.synthetic import synthetic_database
    return [synthetic_database(seed=s) for s in SEEDS]


@pytest.fixture(scope='module')
def tables(dbs):
    return [glue.refiner_views(db, db.get_img_ids(), 128, 6) for db in dbs]


def _subsets(n, rng):
    return {'single': np.array([n - 1]), 'all_sorted': np.arange(n), 'unsorted': rng.permutation(n)[:max(1, n - 2)],
            'reversed': np.arange(n)[::-1].copy(), 'random': rng.permutation(n)[:(n + 1) // 2]}


@pytest.mark.parametrize('n_obj', [1, 3])
def test_refine_rows_equal_object_rows(lib, dbs, tables, n_obj):
    S = 5
    tabs, srcs = tables[:n_obj], [_sources(o, len(t['ids'])) for o, t in enumerate(tables[:n_obj])]
    rng = np.random.RandomState(40 + n_obj)
    Ks = np.stack([dbs[0].K * (1 + 0.01 * s) for s in range(S)], 0)
    Ks[:, 2, 2] = 1
    cams = glue.cameras(Ks)
    n = n_obj * S
    poses = np.concatenate([_random_poses(db, S, 20 + o) for o, db in enumerate(dbs[:n_obj])], 0)
    flags = rng.randint(0, 2, n).astype(np.uint8)
    poses[flags == 1] = poses[flags == 1].astype(np.float32).astype(np.float64)
    want = {f: glue.host_refine_problems_objects(tabs, cams, poses, f, 480, 640, frame_ptr=4096, sources=srcs) for f in (0, 1)}
    for name, idx in _subsets(n, rng).items():
        got = glue.host_refine_problems_rows(tabs, cams, poses, idx, flags, 480, 640, frame_ptr=4096, sources=srcs)
        for j, row in enumerate(idx):
            w = want[int(flags[row])]
            for k in w:
                mine = got[k].reshape(len(idx), -1)[j] if k == 'jobs' else got[k][j]
                theirs = w[k].reshape(n, -1)[row] if k == 'jobs' else w[k][row]
                assert mine.tobytes() == theirs.tobytes(), (name, j, row, k)


@pytest.mark.parametrize('n_obj', [1, 3])
def test_apply_rows_writes_exactly_the_listed_rows(lib, dbs, tables, n_obj):
    S = 4
    tabs = tables[:n_obj]
    rng = np.random.RandomState(60 + n_obj)
    Ks = np.stack([dbs[0].K] * S, 0)
    cams = glue.cameras(Ks)
    n = n_obj * S
    poses = np.concatenate([_random_poses(db, S, 30 + o) for o, db in enumerate(dbs[:n_obj])], 0)
    full = glue.host_refine_problems_objects(tabs, cams, poses, 0, 480, 640)
    net = (rng.randn(n, 7) * 0.05).astype(np.float32)
    net[:, 0] += 1
    want = glue.host_apply_refinements_objects(tabs, full, net)
    canary = np.float64(-12345.678)
    for name, idx in _subsets(n, rng).items():
        prob = {k: np.ascontiguousarray(full[k][idx]) for k in ('que_pose', 'que_K', 'pose_rect')}
        out = np.full((n, 3, 4), canary)
        glue.host_apply_refinements_rows(tabs, prob, net[idx], idx, out)
        listed = np.zeros(n, bool)
        listed[idx] = True
        assert out[listed].tobytes() == want[listed].tobytes(), name
        assert (out[~listed] == canary).all(), name


# ------------------------------------------------------------------------------------------ argument checks
IDX = (C.c_int * 2)(0, 1)
IDX_BAD = {'neg': (C.c_int * 2)(0, -1), 'high': (C.c_int * 2)(0, 6)}          # 3 objects x 2 rows: valid rows 0..5
FLAGS = (C.c_uint8 * 6)()


def _refine_args(views, n_obj=3, rows_per_obj=2, idx=IDX, n_sel=2, flags=FLAGS, cams=BUF, poses=BUF, jobs=BUF):
    return [views, n_obj, rows_per_obj, cams, BUF, 480, 640, poses, idx, n_sel, flags, jobs, BUF, BUF, BUF, BUF, BUF, BUF]


def _apply_args(views, n_obj=3, rows_per_obj=2, idx=IDX, n_sel=2, net_out=BUF, poses=BUF):
    return [views, n_obj, rows_per_obj, BUF, BUF, BUF, net_out, idx, n_sel, poses]


def _bad_cases(tables):
    v3, v17 = _views(tables, 3), _views(tables, 17)
    R, A = 'g6d_glue_refine_problems_rows', 'g6d_glue_apply_refinements_rows'
    return {
        'refine_null_views': (R, _refine_args(None), 'null views'),
        'refine_n_obj_17': (R, _refine_args(v17, n_obj=17), 'n_obj'),
        'refine_rows_0': (R, _refine_args(v3, rows_per_obj=0), 'rows_per_obj'),
        'refine_n_sel_0': (R, _refine_args(v3, n_sel=0), 'n_sel'),
        'refine_null_idx': (R, _refine_args(v3, idx=None), 'n_sel'),
        'refine_null_flags': (R, _refine_args(v3, flags=None), 'bad args'),
        'refine_null_cams': (R, _refine_args(v3, cams=None), 'bad args'),
        'refine_null_poses': (R, _refine_args(v3, poses=None), 'bad args'),
        'refine_null_jobs': (R, _refine_args(v3, jobs=None), 'bad args'),
        'apply_null_views': (A, _apply_args(None), 'null views'),
        'apply_n_obj_0': (A, _apply_args(v3, n_obj=0), 'n_obj'),
        'apply_n_sel_0': (A, _apply_args(v3, n_sel=0), 'n_sel'),
        'apply_null_idx': (A, _apply_args(v3, idx=None), 'n_sel'),
        'apply_null_net_out': (A, _apply_args(v3, net_out=None), 'bad args'),
        'apply_null_poses': (A, _apply_args(v3, poses=None), 'bad args'),
    }


BAD = ['refine_null_views', 'refine_n_obj_17', 'refine_rows_0', 'refine_n_sel_0', 'refine_null_idx', 'refine_null_flags',
       'refine_null_cams', 'refine_null_poses', 'refine_null_jobs', 'apply_null_views', 'apply_n_obj_0', 'apply_n_sel_0',
       'apply_null_idx', 'apply_null_net_out', 'apply_null_poses']


@pytest.mark.parametrize('host', [False, True])
@pytest.mark.parametrize('bad', BAD)
def test_bad_arguments_are_rejected(lib, tables, bad, host):
    name, args, msg = _bad_cases(tables)[bad]
    if host:
        name += '_host'
    else:
        args = args + [None]                                      # the stream
    before = lib.g6d_launch_count()
    assert getattr(lib, name)(*args) == G6D_EINVAL
    err = lib.g6d_last_error()
    assert name.encode() + b':' in err and msg.encode() in err, err
    assert lib.g6d_launch_count() == before


@pytest.mark.parametrize('which', sorted(IDX_BAD))
@pytest.mark.parametrize('entry', ['refine', 'apply'])
def test_host_twins_reject_rows_out_of_range(lib, tables, entry, which):
    v3 = _views(tables, 3)
    if entry == 'refine':
        name, args = 'g6d_glue_refine_problems_rows_host', _refine_args(v3, idx=IDX_BAD[which])
    else:
        name, args = 'g6d_glue_apply_refinements_rows_host', _apply_args(v3, idx=IDX_BAD[which])
    assert getattr(lib, name)(*args) == G6D_EINVAL
    err = lib.g6d_last_error()
    assert name.encode() + b':' in err and b'outside [0, 6)' in err, err


def test_entry_points_are_declared_and_bound():
    for name in ('g6d_glue_refine_problems_rows', 'g6d_glue_apply_refinements_rows'):
        for n in (name, name + '_host'):
            assert n in _lib.header_symbols() and n in _lib._SIGNATURES, n


def test_apply_rows_host_rejects_a_row_listed_twice(lib, tables):
    twice = (C.c_int * 2)(3, 3)
    name = 'g6d_glue_apply_refinements_rows_host'
    assert getattr(lib, name)(*_apply_args(_views(tables, 3), idx=twice)) == G6D_EINVAL
    err = lib.g6d_last_error()
    assert name.encode() + b':' in err and b'listed twice' in err, err
    # building a row's problem twice is allowed (read-only): the same list passes the row checks and the call stops at
    # the null camera pointer instead
    refine = 'g6d_glue_refine_problems_rows_host'
    assert getattr(lib, refine)(*_refine_args(_views(tables, 3), idx=twice, cams=None)) == G6D_EINVAL
    assert b'bad args' in lib.g6d_last_error()


# ------------------------------------------------------------------------------------------ tracker state on the host
def _host_tracker(S=4, num=5):
    from gen6d_b200.track import Tracker
    t = Tracker.__new__(Tracker)               # the state methods only: no estimator, no GPU
    t.S, t.num = S, num
    t.reset()
    return t


def _host_object_tracker(names=('a', 'b'), S=4, num=5):
    from types import SimpleNamespace
    from gen6d_b200.track import ObjectTracker
    t = ObjectTracker.__new__(ObjectTracker)
    t.est = SimpleNamespace(detector=SimpleNamespace(device='cpu'))
    t.names, t.K, t.S, t.num = list(names), len(names), S, num
    t.reset()
    return t


def _poses(n, seed):
    return np.random.RandomState(seed).randn(n, 3, 4)


def test_partial_start_pairs_poses_with_the_listed_sequences():
    t = _host_tracker()
    t._ring[:] = 7
    t._count[:] = 3
    p = _poses(3, 0)
    t.start(p.astype(np.float32), [3, 0, 2])
    q = _poses(1, 1)
    t.start(q, [1])
    for i, s in enumerate([3, 0, 2]):
        np.testing.assert_array_equal(t._prev[s], p[i].astype(np.float32))
    np.testing.assert_array_equal(t._prev[1], q[0])
    assert t._f32.tolist() == [True, False, True, True] and not t._pending.any()
    assert (t._count == 0).all() and (t._ring == 0).all()
    t._count[:] = 3
    t.reset([2, 0])
    assert t._pending.tolist() == [True, False, True, False] and t._count.tolist() == [0, 3, 0, 3]


def test_object_tracker_partial_start_pairs_poses_with_the_listed_sequences():
    t = _host_object_tracker()
    t._count[:] = 3
    pa, pb = _poses(2, 2), _poses(2, 3)
    t.start({'a': pa, 'b': pb}, [3, 1])
    prev = t._prev.numpy().reshape(2, 4, 3, 4)
    np.testing.assert_array_equal(prev[0, 3], pa[0])
    np.testing.assert_array_equal(prev[0, 1], pa[1])
    np.testing.assert_array_equal(prev[1, 3], pb[0])
    np.testing.assert_array_equal(prev[1, 1], pb[1])
    assert t._count.tolist() == [3, 0, 3, 0, 3, 0, 3, 0] and t._f32.tolist() == [True, False, True, False]


@pytest.mark.parametrize('bad', [[4], [-1], [1, 1]])
def test_sequences_are_validated(bad):
    t = _host_tracker()
    with pytest.raises(ValueError):
        t.reset(bad)
    with pytest.raises(ValueError):
        t.start(np.zeros((len(bad), 3, 4)), bad)
    with pytest.raises(ValueError):
        t.start(np.zeros((2, 3, 4)), [1])


@pytest.mark.parametrize('F,r', [(3, 1), (1, 3), (2, 2), (1, 1)])
@pytest.mark.parametrize('K', [1, 3])
def test_mixed_plan_padding_never_targets_a_real_row(K, F, r):
    """Every subset of every size at S = 7: the padding slots scatter into scratch rows only, each iteration lists exactly
    the real rows whose chain is still running (ascending, then scratch rows), and the shapes depend on the bucket only."""
    from itertools import combinations
    from gen6d_b200.track import _bucket, _iter_lengths, _mixed_inputs
    S = 7
    f32 = np.ones(S, bool)
    shapes = {}
    for m in range(0, S):
        for reinit in combinations(range(S), m):
            pending = np.zeros(S, bool)
            pending[list(reinit)] = True
            got, b, (seq, tgt, flags, lists) = _mixed_inputs(S, K, pending, f32, F, r, 'cpu')
            n = S + b
            assert b == _bucket(m, S) and got.tolist() == list(reinit)
            assert seq.tolist()[:m] == list(reinit) and set(seq.tolist()[m:]) <= set(reinit)
            tgt = tgt.numpy().reshape(K, b) - np.arange(K)[:, None] * n
            assert (tgt[:, :m] == np.asarray(reinit)).all() and (tgt[:, m:] >= S).all()
            lists, off = lists.numpy(), 0
            for it, L in enumerate(_iter_lengths(S, b, F, r)):
                running = [s for s in range(S) if (s in reinit and it < F) or (s not in reinit and it < r)]
                for o in range(K):
                    rows = lists[off:off + L] - o * n
                    off += L
                    assert rows[rows < S].tolist() == running and (np.diff(rows) > 0).all()
            assert off == len(lists)
            shapes.setdefault(b, set()).add((tuple(seq.shape), tuple(tgt.shape), tuple(flags.shape), tuple(lists.shape)))
    assert all(len(v) == 1 for v in shapes.values()), shapes
