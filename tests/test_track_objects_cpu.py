"""The object-indexed refinement glue and smoothing (g6d_glue_refine_problems_objects, g6d_glue_apply_refinements_objects,
g6d_track_smooth_objects) through their *_host twins, without a GPU: every row of an object set must be bit-identical to
the single-object entry point called on that object's slice, and bad arguments must be rejected before any launch."""
import ctypes as C

import numpy as np
import pytest

from gen6d_b200 import _lib, glue
from gen6d_b200 import track as T

G6D_EINVAL = -1
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


def _sources(o, nv):
    return (10 ** 9 * (o + 1) + 7 * np.arange(nv), np.full(nv, 480 + o), np.full(nv, 640 - o))


def _random_poses(db, n, seed):
    ids = db.get_img_ids()
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        p = db.get_pose(ids[rng.randint(len(ids))]).astype(np.float64).copy()
        w = rng.randn(3) * 0.05
        Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        U, _, Vt = np.linalg.svd((np.eye(3) + Wx) @ p[:, :3])
        p[:, :3] = U @ Vt
        p[:, 3] += rng.randn(3) * 0.02
        out.append(p)
    return np.stack(out, 0)


@pytest.mark.parametrize('f32', [0, 1])
@pytest.mark.parametrize('S', [1, 4])
def test_glue_objects_equal_per_object_calls(lib, dbs, tables, S, f32):
    K = len(tables)
    rng = np.random.RandomState(100 * S + f32)
    Ks = np.stack([dbs[0].K * (1 + 0.01 * s) for s in range(S)], 0)
    Ks[:, 2, 2] = 1
    cams = glue.cameras(Ks)
    poses = np.concatenate([_random_poses(db, S, 10 + o) for o, db in enumerate(dbs)], 0)
    if f32:
        poses = poses.astype(np.float32).astype(np.float64)
    sources = [_sources(o, len(t['ids'])) for o, t in enumerate(tables)]
    got = glue.host_refine_problems_objects(tables, cams, poses, f32, 480, 640, frame_ptr=4096, sources=sources)
    net = (rng.randn(K * S, 7) * 0.05).astype(np.float32)
    net[:, 0] += 1
    got_poses = glue.host_apply_refinements_objects(tables, got, net)
    for o in range(K):
        r = slice(o * S, (o + 1) * S)
        src, img_rows, img_cols = sources[o]
        want = glue.host_refine_problems(tables[o], cams, poses[r], f32, 480, 640, frame_ptr=4096, src=src, img_rows=img_rows,
                                         img_cols=img_cols)
        for k in want:
            mine = got[k].reshape(K * S, -1)[r] if k == 'jobs' else got[k][r]
            theirs = want[k].reshape(S, -1) if k == 'jobs' else want[k]
            assert mine.tobytes() == theirs.tobytes(), (o, k)
        prob = {k: np.ascontiguousarray(got[k][r]) for k in ('que_pose', 'que_K', 'pose_rect')}
        want_poses = glue.host_apply_refinements(tables[o], prob, net[r])
        assert got_poses[r].tobytes() == want_poses.tobytes(), o
    # the frame part reads frame s of the shared frames, whatever the object
    jobs = got['jobs'].reshape(K, S, -1)
    for s in range(S):
        assert (jobs['src'][:, s, 0] == 4096 + s * 480 * 640 * 3).all()


@pytest.mark.parametrize('f32', [False, True])
@pytest.mark.parametrize('S', [1, 4])
def test_smoothing_objects_equal_per_object_calls(lib, S, f32):
    from golden import track_cases
    K, num, L = 3, 4, 6
    cases = [[track_cases.smoothing_case(seed=700 + 10 * o + s, L=L) for s in range(S)] for o in range(K)]
    bboxes = np.stack([T.bbox_from_points(cases[o][0]['pts']) for o in range(K)], 0)
    Ks = np.stack([cases[0][s]['K'] for s in range(S)], 0)
    w = T.smoothing_weights(num, 2.5)
    ring, count = np.zeros((K * S, num, 8, 2), np.float32), np.zeros(K * S, np.int32)
    rings = [np.zeros((S, num, 8, 2), np.float32) for _ in range(K)]
    counts = [np.zeros(S, np.int32) for _ in range(K)]
    for k in range(L):
        poses = np.stack([cases[o][s]['poses'][k] for o in range(K) for s in range(S)], 0).astype(np.float64)
        if f32:
            poses = poses.astype(np.float32).astype(np.float64)
        sm, avg = T.host_smooth_objects(poses, f32, bboxes, Ks, ring, count, w)
        for o in range(K):
            r = slice(o * S, (o + 1) * S)
            sm_o, avg_o = T.host_smooth(poses[r], f32, bboxes[o], Ks, rings[o], counts[o], w)
            assert sm[r].tobytes() == sm_o.tobytes() and avg[r].tobytes() == avg_o.tobytes(), (k, o)
            assert ring[r].tobytes() == rings[o].tobytes() and count[r].tobytes() == counts[o].tobytes(), (k, o)
    assert (count == min(L, num)).all()


# ------------------------------------------------------------------------------------------ argument checks
BUF = C.c_void_p(16)            # never dereferenced: every call below is rejected before a launch


def _views(tables, n, ref_num=None):
    ts = [tables[o % len(tables)] for o in range(n)]
    out = (_lib.GlueViews * max(n, 1))(*[glue.views_struct({k: 16 for k in ('poses', 'R_look', 'RlookR', 'f', 'Kinv', 'even_idx',
                                                                             'even_dirs')}, t, 16, 16, 16) for t in ts])
    if ref_num is not None:
        out[n - 1].ref_num = ref_num
    return out


def _refine_args(views, n_obj=3, rows_per_obj=2, cams=BUF, poses=BUF, jobs=BUF):
    return [views, n_obj, rows_per_obj, cams, BUF, 480, 640, poses, 1, jobs, BUF, BUF, BUF, BUF, BUF, BUF]


def _apply_args(views, n_obj=3, rows_per_obj=2, net_out=BUF, poses=BUF):
    return [views, n_obj, rows_per_obj, BUF, BUF, BUF, net_out, poses]


def _smooth_args(n_obj=3, rows_per_obj=2, poses=BUF, bboxes=BUF, Ks=BUF, num=5):
    return [poses, 1, bboxes, n_obj, rows_per_obj, Ks, BUF, BUF, num, BUF, BUF, BUF]


def _bad_cases(tables):
    v3, v17 = _views(tables, 3), _views(tables, 17)
    return {
        'refine_null_views': ('g6d_glue_refine_problems_objects', _refine_args(None), 'null views'),
        'refine_n_obj_0': ('g6d_glue_refine_problems_objects', _refine_args(v3, n_obj=0), 'n_obj'),
        'refine_n_obj_17': ('g6d_glue_refine_problems_objects', _refine_args(v17, n_obj=17), 'n_obj'),
        'refine_rows_0': ('g6d_glue_refine_problems_objects', _refine_args(v3, rows_per_obj=0), 'rows_per_obj'),
        'refine_ref_num': ('g6d_glue_refine_problems_objects', _refine_args(_views(tables, 3, ref_num=5)), 'same'),
        'refine_null_cams': ('g6d_glue_refine_problems_objects', _refine_args(v3, cams=None), 'bad args'),
        'refine_null_poses': ('g6d_glue_refine_problems_objects', _refine_args(v3, poses=None), 'bad args'),
        'refine_null_jobs': ('g6d_glue_refine_problems_objects', _refine_args(v3, jobs=None), 'bad args'),
        'apply_null_views': ('g6d_glue_apply_refinements_objects', _apply_args(None), 'null views'),
        'apply_n_obj_0': ('g6d_glue_apply_refinements_objects', _apply_args(v3, n_obj=0), 'n_obj'),
        'apply_n_obj_17': ('g6d_glue_apply_refinements_objects', _apply_args(v17, n_obj=17), 'n_obj'),
        'apply_rows_0': ('g6d_glue_apply_refinements_objects', _apply_args(v3, rows_per_obj=0), 'rows_per_obj'),
        'apply_null_net_out': ('g6d_glue_apply_refinements_objects', _apply_args(v3, net_out=None), 'bad args'),
        'apply_null_poses': ('g6d_glue_apply_refinements_objects', _apply_args(v3, poses=None), 'bad args'),
        'smooth_n_obj_0': ('g6d_track_smooth_objects', _smooth_args(n_obj=0), 'n_obj'),
        'smooth_rows_0': ('g6d_track_smooth_objects', _smooth_args(rows_per_obj=0), 'rows_per_obj'),
        'smooth_num_0': ('g6d_track_smooth_objects', _smooth_args(num=0), 'num'),
        'smooth_null_poses': ('g6d_track_smooth_objects', _smooth_args(poses=None), 'null pointer'),
        'smooth_null_bboxes': ('g6d_track_smooth_objects', _smooth_args(bboxes=None), 'null pointer'),
        'smooth_null_Ks': ('g6d_track_smooth_objects', _smooth_args(Ks=None), 'null pointer'),
    }


BAD = sorted(['refine_null_views', 'refine_n_obj_0', 'refine_n_obj_17', 'refine_rows_0', 'refine_ref_num', 'refine_null_cams',
              'refine_null_poses', 'refine_null_jobs', 'apply_null_views', 'apply_n_obj_0', 'apply_n_obj_17', 'apply_rows_0',
              'apply_null_net_out', 'apply_null_poses', 'smooth_n_obj_0', 'smooth_rows_0', 'smooth_num_0', 'smooth_null_poses',
              'smooth_null_bboxes', 'smooth_null_Ks'])


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


def test_views_fit_the_parameter_block():
    assert C.sizeof(_lib.GlueViews) == 120
    assert _lib.G6D_GLUE_MAX_OBJECTS * C.sizeof(_lib.GlueViews) < 4096


def test_entry_points_are_declared_and_bound():
    for name in ('g6d_glue_refine_problems_objects', 'g6d_glue_apply_refinements_objects', 'g6d_track_smooth_objects'):
        for n in (name, name + '_host'):
            assert n in _lib.header_symbols() and n in _lib._SIGNATURES, n
    header = open(_lib.HEADER_PATH).read()
    assert f'#define G6D_GLUE_MAX_OBJECTS {_lib.G6D_GLUE_MAX_OBJECTS}' in header
