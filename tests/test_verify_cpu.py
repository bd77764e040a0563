"""Checking tracked poses with the detector (row f20) without a GPU: the g6d_verify_windows / g6d_verify_judge host twins
(the code the kernels run) against the numpy restatement in verify_oracle.py, bit for bit; the window record as the
inverse of poses_from_similarity; and the trackers' verification schedule, names and argument checks."""
import types

import numpy as np
import pytest

import verify_oracle as oracle
from golden import cases
from gen6d_b200 import _lib, geometry as G, glue, verify as V
from gen6d_b200.database import SyntheticObjectDatabase


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()
    return _lib.lib()


@pytest.fixture(scope='module')
def db():
    return SyntheticObjectDatabase(**cases.estimator_case()['db'])


def refs_of(db, n_views, seed):
    ids = [str(i) for i in G.select_views_fps(db, db.get_img_ids(), n_views)]
    _, ref_Ks, ref_poses, _ = G.normalize_reference_views(db, ids, 128, 0.05, warp=False)
    info = {'poses': ref_poses, 'Ks': ref_Ks, 'center': db.object_center() + np.random.RandomState(seed).randn(3) * 0.01 * seed}
    return info, glue.selector_refs(info)


def random_Ks(rng, n):
    Ks = []
    for i in range(n):
        f = 400 + rng.rand() * 400
        K = np.asarray([[f, 0, 300 + rng.rand() * 40], [0, f * (0.9 + 0.2 * rng.rand()), 220 + rng.rand() * 40], [0, 0, 1]])
        Ks.append(K.astype(np.float32 if i % 2 else np.float64))
    return Ks


def random_poses(db, rng, n):
    ids = db.get_img_ids()
    out = []
    for _ in range(n):
        p = db.get_pose(ids[rng.randint(len(ids))]).astype(np.float64).copy()
        w = rng.randn(3) * 0.1
        Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        U, _, Vt = np.linalg.svd((np.eye(3) + Wx) @ p[:, :3])
        p[:, :3] = U @ Vt
        p[:, 3] += rng.randn(3) * 0.05
        out.append(p)
    return np.stack(out, 0)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------------------------------ windows
@pytest.mark.parametrize('K_obj', [1, 3])
@pytest.mark.parametrize('f32', [False, True])
def test_windows_equal_the_oracle(lib, db, K_obj, f32):
    rng = np.random.RandomState(3 * K_obj + f32)
    qn = 7
    refs = [refs_of(db, 8 + 4 * o, o)[1] for o in range(K_obj)]
    cams = np.concatenate([glue.cameras(K[None]) for K in random_Ks(rng, qn)], 0)    # float32 and float64 intrinsics
    poses = random_poses(db, rng, K_obj * qn)
    poses[1, :, 3] *= -1                                              # the object behind the camera
    poses[2, 2, 3] = 0.0                                              # the centre at depth ~0
    poses[3, 0, 0] = np.nan
    poses[4, 1, 3] = np.inf
    poses[5, :, :] = 0.0                                              # camera at the object centre: que_dist 0
    if f32:
        poses = poses.astype(np.float32)
    got = V.host_windows(poses, f32, refs, cams)
    want = oracle.windows(poses, f32, refs, cams)
    assert same(got, want), np.flatnonzero((got != want).any(1))
    assert (got[[1, 3, 4, 5], 3] == 0).all() and (got[[1, 3, 4, 5]] == [0, 0, 1, 0]).all()
    assert got[0, 3] == 1 and got[6, 3] == 1


def test_float32_flag_reads_rounded_values(lib, db):
    rng = np.random.RandomState(11)
    _, refs = refs_of(db, 8, 0)
    cams = glue.cameras(np.stack([db.K] * 4, 0))
    poses = random_poses(db, rng, 4) + rng.randn(4, 3, 4) * 1e-9
    assert same(V.host_windows(poses, True, [refs], cams), V.host_windows(poses.astype(np.float32), True, [refs], cams))
    assert same(V.host_windows(poses, False, [refs], cams), oracle.windows(poses, False, [refs], cams))


def test_windows_invert_poses_from_similarity(lib, db):
    """detection -> poses_from_similarity (random angles and reference views) -> window record: (x, y, scale) again."""
    rng = np.random.RandomState(5)
    info, refs = refs_of(db, 16, 0)
    n = 64
    det = np.stack([200 + rng.rand(n) * 240, 150 + rng.rand(n) * 180, 0.4 + rng.rand(n) * 1.6], 1).astype(np.float32)
    ang = (rng.rand(n) * 2 * np.pi - np.pi).astype(np.float32)
    idx = rng.randint(0, len(info['poses']), n)
    for K in (db.K, db.K.astype(np.float64)):
        Ks = np.stack([K] * n, 0)
        poses = G.poses_from_similarity(det[:, :2], det[:, 2], ang, info['poses'][idx], info['Ks'][idx], Ks, info['center'])
        for f32 in (False, True):
            rec = V.host_windows(poses.astype(np.float32) if f32 else poses, f32, [refs], glue.cameras(Ks))
            assert (rec[:, 3] == 1).all()
            np.testing.assert_allclose(rec[:, :3], det, rtol=1e-5)


# ------------------------------------------------------------------------------------------ judge
def judge_problem(rng, n=40):
    rec = np.stack([rng.rand(n) * 640, rng.rand(n) * 480, 0.3 + rng.rand(n) * 2, np.ones(n)], 1).astype(np.float32)
    rec[::7] = [0, 0, 1, 0]                                           # invalid records
    det = np.stack([rng.rand(n) * 256, rng.rand(n) * 256, 0.2 + rng.rand(n) * 3, rng.randn(n)], 1).astype(np.float32)
    det[3, 3] = np.nan
    det[5, 3] = -np.inf
    det[6, :2] = np.nan
    return rec, det


@pytest.mark.parametrize('thr', [(None, None), (0.0, None), (None, 0.25), (-0.5, 0.4), (np.inf, None), (-np.inf, 0.0)])
def test_judge_equals_the_oracle(lib, thr):
    rec, det = judge_problem(np.random.RandomState(2))
    got = V.host_judge(rec, det, 256, 128, *thr)
    want = oracle.judge(rec, det, 256, 128, *thr)
    assert same(got[0], want[0]) and same(got[1], want[1])
    assert got[1][::7].all()                                          # invalid records are always lost
    if thr[0] is not None:
        assert got[1][3] == 1                                         # a NaN score is lost
    if thr[1] is not None:
        assert got[1][6] == 1                                         # a NaN offset is lost


def test_judge_maps_back_and_keeps_ties(lib):
    rng = np.random.RandomState(4)
    rec, det = judge_problem(rng)
    out, _ = V.host_judge(rec, det, 256, 128)
    ok = np.isfinite(det[:, :2]).all(1)
    np.testing.assert_allclose(out[ok, :2], rec[ok, :2] + (det[ok, :2] - 128) * rec[ok, 2:3], rtol=1e-6, atol=1e-3)
    np.testing.assert_allclose(out[:, 2], det[:, 2] * rec[:, 2], rtol=1e-6)
    # thresholds equal to a row's reported score / offset keep that row
    i = 1
    _, lost = V.host_judge(rec, det, 256, 128, float(out[i, 3]), float(out[i, 4]))
    assert lost[i] == 0
    _, lost = V.host_judge(rec, det, 256, 128, float(np.nextafter(out[i, 3], np.float32(np.inf))), None)
    assert lost[i] == 1
    _, lost = V.host_judge(rec, det, 256, 128, None, float(np.nextafter(out[i, 4], np.float32(0))))
    assert lost[i] == 1


def test_entry_points_reject_bad_arguments(lib, db):
    _, refs = refs_of(db, 8, 0)
    cams = glue.cameras(np.stack([db.K] * 2, 0))
    with pytest.raises(_lib.Gen6DLibraryError, match='n_obj'):
        V.host_windows(np.zeros((0, 3, 4)), False, [], cams)
    with pytest.raises(ValueError):
        V.host_windows(np.zeros((3, 3, 4)), False, [refs], cams)
    rec, det = judge_problem(np.random.RandomState(0), 8)
    with pytest.raises(_lib.Gen6DLibraryError, match='NaN'):
        V.host_judge(rec, det, 256, 128, np.nan, None)
    with pytest.raises(_lib.Gen6DLibraryError, match='window'):
        V.host_judge(rec, det, 0, 128)


def test_entry_points_are_declared_and_bound():
    names = {'g6d_verify_windows', 'g6d_verify_windows_host', 'g6d_verify_judge', 'g6d_verify_judge_host'}
    assert names <= set(_lib.header_symbols())
    assert names <= set(_lib._SIGNATURES)


# ------------------------------------------------------------------------------------------ the schedule
def run_schedule(every, kinds, S=1):
    """kinds: per step 'full', 'refine' or 'mixed:<reinit seqs>' over all S sequences -> the steps that verify."""
    sch, since = V.Schedule(every), np.zeros(S, np.int64)
    out = []
    for t, kind in enumerate(kinds):
        seqs = np.arange(S)
        pending = np.full(S, kind == 'full')
        if kind.startswith('mixed'):
            pending[[int(v) for v in kind.split(':')[1].split(',')]] = True
            kind = 'mixed'
        check = sch.due(kind, since[seqs])
        sch.advance(since, seqs, pending, check)
        if check:
            out.append(t)
    return out


@pytest.mark.parametrize('every', range(1, 7))
def test_which_steps_verify(every):
    kinds = ['full'] + ['refine'] * 20
    assert run_schedule(every, kinds) == list(range(every, 21, every))
    # a full prediction restarts the count; a mixed step counts its refining rows but never verifies
    kinds = ['full'] + ['refine'] * 3 + ['full'] + ['refine'] * 8
    want = [t for t in range(1, 4) if t % every == 0] + [4 + t for t in range(1, 9) if t % every == 0]
    assert run_schedule(every, kinds) == want
    kinds = ['full'] + ['refine'] * (every - 1) + ['mixed:1'] + ['refine'] * 3
    assert run_schedule(every, kinds, S=2) == [every + 1] + [every + 1 + t for t in range(1, 3) if t % every == 0]
    assert run_schedule(None, ['full'] + ['refine'] * 10) == []


def test_counts_under_partial_steps_and_restarts():
    sch, since = V.Schedule(3), np.zeros(4, np.int64)
    all4 = np.arange(4)
    sch.advance(since, all4, np.ones(4, bool), False)                 # full
    for _ in range(2):
        assert not sch.due('refine', since)
        sch.advance(since, all4, np.zeros(4, bool), False)
    assert since.tolist() == [2, 2, 2, 2]
    since[1] = 0                                                       # reset([1]) / start(poses, [1])
    assert sch.due('refine', since[[1, 2]])                            # sequence 2 reaches 3: both are verified
    sch.advance(since, np.asarray([1, 2]), np.zeros(2, bool), True)
    assert since.tolist() == [2, 0, 0, 2]
    assert not sch.due('refine', since[[1]])
    assert not sch.due('full', since) and not sch.due('mixed', since)
    sch.advance(since, all4, np.asarray([True, False, False, False]), False)   # mixed: 0 re-initialised, the others count
    assert since.tolist() == [0, 1, 1, 3]
    assert sch.due('refine', since[[3]])


def fake_estimator():
    det = types.SimpleNamespace(device='cpu')
    return types.SimpleNamespace(refiner=object(), detector=det, cfg={'refine_iter': 1, 'device_glue': False, 'host_warps': False},
                                 _generation=lambda: (0,), _glue_possible=lambda: False)


def box():
    return np.asarray([[x, y, z] for z in (-1, 1) for x, y in ((-1, -1), (-1, 1), (1, 1), (1, -1))], np.float32)


def test_tracker_counts_and_lost_sequences_become_pending():
    from gen6d_b200.track import Tracker
    trk = Tracker(fake_estimator(), 4, bbox_3d=box(), verify_every=2, lost_score=0.5)
    trk._pending[:] = False
    trk._since[:] = [1, 1, 1, 1]
    trk.start(np.tile(np.eye(3, 4), (1, 1, 1)), [2])
    assert trk._since.tolist() == [1, 1, 0, 1]
    lost = trk._verify.lost_sequences(np.asarray([3, 0, 1]), np.asarray([True, False, True]))
    assert lost.tolist() == [3, 1]
    trk.reset(lost)
    assert trk._pending.tolist() == [False, True, False, True]
    assert trk._since.tolist() == [1, 0, 0, 0]
    trk.reset()
    assert trk._pending.all() and (trk._since == 0).all()
    # thresholds None: verify and report, never reset
    quiet = Tracker(fake_estimator(), 2, bbox_3d=box(), verify_every=1)
    assert quiet._verify.lost_sequences(np.arange(2), np.ones(2, bool)).tolist() == []


def test_verification_needs_the_device_pipeline():
    from gen6d_b200.track import Tracker
    trk = Tracker(fake_estimator(), 1, bbox_3d=box(), verify_every=1)
    with pytest.raises(ValueError, match='verify_every'):
        trk.step([np.zeros((8, 8, 3), np.uint8)], [np.eye(3)])


def test_graph_names_are_apart():
    from gen6d_b200 import frames as fr
    from gen6d_b200.track import PartialStep
    plan = fr.FramePlan([(48, 64), (40, 56)])
    part = PartialStep(8, 1, [0, 3, 5], np.zeros(8, bool), np.ones(8, bool), 1)
    wraps = [lambda n: n, part.name, lambda n: (n, 'draw', ('raw',)), plan.key, plan.device_key,
             lambda n: plan.device_key(n, True), lambda n: plan.key(part.name((n, 'draw', ('raw', 'smoothed'))))]
    plain = {'track_full', 'track_refine0', 'track_refine1', 'track_mixed1', 'track_mixed4', 'predict', 'verify_poses',
             ('instances', 4, 1, 0.3, None)}
    keys = [(None, None), (0.5, None), (None, 0.25), (np.inf, 1.0)]
    verifying = {w(V.graph_name(b, k)) for w in wraps for b in ('track_refine0', 'track_refine1') for k in keys}
    existing = {w(b) for w in wraps for b in plain}
    assert len(verifying) == len(wraps) * 2 * len(keys)
    assert not verifying & existing


def test_argument_errors():
    for bad in (0, -1, 1.5, 'x', True):
        with pytest.raises(ValueError, match='verify_every'):
            V.Schedule(bad)
    with pytest.raises(ValueError, match='verify_every too'):
        V.Schedule(None, lost_score=0.0)
    with pytest.raises(ValueError, match='verify_every too'):
        V.Schedule(None, lost_gate=0.5)
    with pytest.raises(ValueError, match='NaN'):
        V.Schedule(1, lost_score=float('nan'))
    with pytest.raises(ValueError, match='lost_gate'):
        V.Schedule(1, lost_gate=-0.1)
    with pytest.raises(ValueError, match='number'):
        V.check_thresholds('high', None)
    assert V.check_thresholds(1, np.float32(0.5)) == (1.0, 0.5)
    from gen6d_b200.track import Tracker
    with pytest.raises(ValueError, match='verify_every'):
        Tracker(fake_estimator(), 2, bbox_3d=box(), verify_every=0)
