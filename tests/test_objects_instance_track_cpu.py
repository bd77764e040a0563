"""The object set's association (g6d_instances_associate_objects_host: the code the device kernel runs) against K chained
single-object calls (g6d_instances_associate_host on each object's slice, the id counter passed from call to call), bit
for bit on every output and state array, plus its argument checks.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from tests.test_instance_track_cpu import NUM, OUTS, STATE, _project, make_problem

G6D_EINVAL = -1


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200 import _lib
    from gen6d_b200.build import build
    build()
    return _lib.lib()


def make_set_problem(rng, K, S=None, M=None, F=None, r=None):
    """K objects' make_problem()s on shared cameras, gate, max_misses and counter, laid out in the set's slot-major rows
    (row (m*K + o)*S + s).  Objects after the first get detections placed near their own tracks' projections with the
    shared cameras, so every object matches, spawns and drops."""
    p0 = make_problem(rng, S=S, M=M, F=F, r=r)
    S, M = len(p0['cams']), len(p0['live']) // len(p0['cams'])
    objs = [p0]
    for _ in range(1, K):
        p = make_problem(rng, S=S, M=M, F=p0['F'], r=p0['r'])
        p['cams'] = p0['cams']
        for i in range(M * S):
            s, t = i % S, rng.randint(M) * S + i % S
            if rng.rand() < 0.7 and p['prev'][t].reshape(3, 4)[2, 3] > 0:
                xy = _project(p['prev'][t].reshape(3, 4), p0['cams'][s, :9].reshape(3, 3), p['center'])
                p['det'][i, :2] = xy + rng.randn(2) * rng.choice([1, 10, 60])
        objs.append(p)
    rows = lambda o: np.asarray([(m * K + o) * S + s for m in range(M) for s in range(S)])
    full = {k: p0[k] for k in ('cams', 'res', 'gate', 'max_misses', 'F', 'r', 'next_id')}
    full['centers'] = np.stack([p['center'] for p in objs], 0)
    for k in ('det', 'valid', 'init', 'prev', 'live', 'ids', 'misses', 'park', 'ring', 'count'):
        a = np.zeros((M * K * S,) + p0[k].shape[1:], p0[k].dtype)
        for o, p in enumerate(objs):
            a[rows(o)] = p[k]
        full[k] = a
    return full, K, S, M


ARGS = ('det', 'valid', 'init', 'cams', 'centers', 'res', 'gate', 'max_misses', 'F', 'r', 'prev')


def run_set(p):
    from gen6d_b200.instance_track import host_associate_objects
    q = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
    outs = host_associate_objects(*[q[k] for k in ARGS], *[q[k] for k in STATE])
    return {**dict(zip(OUTS, outs)), **{k: q[k] for k in STATE}}


def run_chained(p, K, S, M):
    """K g6d_instances_associate_host calls on the objects' slices, in object order, continuing the counter; the slices'
    results scattered back to the set's rows (work rows and list entries remapped to the set's work layout)."""
    from gen6d_b200.instance_track import host_associate
    q = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
    n, n_it = M * K * S, max(p['F'], p['r'])
    out = {'work': np.zeros((2 * n, 12)), 'flags0': np.zeros(2 * n, np.uint8), 'lists': np.zeros(n_it * n, np.int32),
           'det_slot': np.zeros(n, np.int32), 'spawned': np.zeros(n, np.int32), 'dropped': np.zeros(n, np.int64)}
    next_id = q['next_id']
    for o in range(K):
        rows = np.asarray([(m * K + o) * S + s for m in range(M) for s in range(S)])
        wrows = np.asarray([(m * K + o) * 2 * S + x for m in range(M) for x in range(2 * S)])
        sl = {k: np.ascontiguousarray(q[k][rows]) for k in ('det', 'valid', 'init', 'prev', 'live', 'ids', 'misses', 'park', 'ring',
                                                            'count')}
        work, flags0, lists, det_slot, spawned, dropped = host_associate(
            sl['det'], sl['valid'], sl['init'], q['cams'], q['centers'][o], q['res'], q['gate'], q['max_misses'], q['F'], q['r'],
            sl['prev'], sl['live'], sl['ids'], sl['misses'], next_id, sl['park'], sl['ring'], sl['count'])
        for k in ('live', 'ids', 'misses', 'park', 'ring', 'count'):
            q[k][rows] = sl[k]
        out['work'][wrows], out['flags0'][wrows] = work, flags0
        out['det_slot'][rows], out['spawned'][rows], out['dropped'][rows] = det_slot, spawned, dropped
        for it in range(n_it):
            out['lists'][it * n + rows] = wrows[lists[it * M * S:(it + 1) * M * S]]
    return {**out, **{k: q[k] for k in STATE}}


def assert_same(got, want, tag=''):
    for k in OUTS + STATE:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.shape == w.shape and g.dtype == w.dtype, (tag, k, g.shape, w.shape, g.dtype, w.dtype)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), (tag, k, g, w)


@pytest.mark.parametrize('K', [1, 2, 3, 5])
def test_random_problems_equal_chained_single_object_calls(lib, K):
    rng = np.random.RandomState(100 + K)
    n_match = n_spawn = n_drop = 0
    for trial in range(400):
        p, K_, S, M = make_set_problem(rng, K)
        got, want = run_set(p), run_chained(p, K_, S, M)
        assert_same(got, want, trial)
        n_spawn += int(got['spawned'].sum())
        n_drop += int((got['dropped'] >= 0).sum())
        n_match += int(((got['det_slot'] >= 0) & (p['valid'] != 0)).sum()) - int(got['spawned'].sum())
    assert min(n_match, n_spawn, n_drop) > 50, (n_match, n_spawn, n_drop)


def test_ids_in_object_sequence_detection_order(lib):
    """No live tracks and every detection valid: the ids run over (object, sequence, detection) in that order."""
    rng = np.random.RandomState(5)
    K, S, M = 3, 2, 2
    p, *_ = make_set_problem(rng, K, S=S, M=M, F=1, r=1)
    p['live'][:], p['ids'][:], p['valid'][:], p['next_id'][:] = 0, -1, 1, 40
    got = run_set(p)
    assert got['spawned'].all() and got['next_id'][0] == 40 + M * K * S
    for o in range(K):
        for s in range(S):
            for m in range(M):
                assert got['ids'][(m * K + o) * S + s] == 40 + (o * S + s) * M + m


def test_single_object_equals_single_object_call(lib):
    from tests.test_instance_track_cpu import run_both
    rng = np.random.RandomState(77)
    for trial in range(300):
        p = make_problem(rng)
        want, _ = run_both(p)
        q = {**p, 'centers': np.asarray(p['center'], np.float64).reshape(1, 3)}
        assert_same(run_set(q), want, trial)


def test_many_pairs(lib):
    """K*S beyond one CTA's 256 threads: the device scan runs chunked; the host twin must still equal the chain."""
    rng = np.random.RandomState(9)
    p, K, S, M = make_set_problem(rng, 5, S=60, M=2, F=2, r=1)
    assert_same(run_set(p), run_chained(p, K, S, M))


def _raw_args(p, K, S, M, /, **over):
    a = {k: (np.ascontiguousarray(v) if isinstance(v, np.ndarray) else v) for k, v in p.items()}
    n, n_it = M * K * S, max(p['F'], p['r'])
    bufs = {'work': np.zeros((2 * n, 12)), 'flags0': np.zeros(2 * n, np.uint8), 'lists': np.zeros(n_it * n, np.int32),
            'det_slot': np.zeros(n, np.int32), 'spawned': np.zeros(n, np.int32), 'dropped': np.zeros(n, np.int64)}
    a.update(bufs)
    ptr = lambda k: None if over.get(k, 0) is None else a[k].ctypes.data
    val = lambda k, v: over.get(k, v)
    args = [val('S', S), val('K', K), val('M', M), a['F'], a['r'], ptr('det'), ptr('valid'), ptr('init'), ptr('cams'), ptr('centers'),
            a['res'], val('gate', a['gate']), val('max_misses', a['max_misses']), ptr('prev'), ptr('live'), ptr('ids'), ptr('misses'),
            ptr('next_id'), ptr('park'), ptr('ring'), ptr('count'), NUM, ptr('work'), ptr('flags0'), ptr('lists'), ptr('det_slot'),
            ptr('spawned'), ptr('dropped')]
    return args, a


BAD = {'K_0': (dict(K=0), 'K >= 1'), 'M_0': (dict(M=0), 'M <= 16'), 'M_17': (dict(M=17), 'M <= 16'),
       'S_0': (dict(S=0), 'S >= 1'), 'null_centers': (dict(centers=None), 'null pointer (centers)'),
       'null_det': (dict(det=None), 'null pointer'), 'null_next_id': (dict(next_id=None), 'null pointer'),
       'gate_0': (dict(gate=0.0), 'gate'), 'max_misses_neg': (dict(max_misses=-1), 'max_misses')}


@pytest.mark.parametrize('host', [False, True])
@pytest.mark.parametrize('bad', sorted(BAD))
def test_bad_arguments_are_rejected(lib, bad, host):
    p, K, S, M = make_set_problem(np.random.RandomState(3), 2, S=2, M=2, F=1, r=1)
    over, msg = BAD[bad]
    args, a = _raw_args(p, K, S, M, **over)
    name = 'g6d_instances_associate_objects' + ('_host' if host else '')
    if not host:
        args = args + [None]                                      # the stream
    live = a['live'].copy()
    before = lib.g6d_launch_count()
    assert getattr(lib, name)(*args) == G6D_EINVAL
    err = lib.g6d_last_error()
    assert name.encode() + b':' in err and msg.encode() in err, err
    assert lib.g6d_launch_count() == before
    np.testing.assert_array_equal(a['live'], live)               # nothing was touched


def test_numpy_wrapper_checks(lib):
    from gen6d_b200 import _lib
    p, K, S, M = make_set_problem(np.random.RandomState(4), 2, S=2, M=2, F=1, r=1)
    with pytest.raises(ValueError):                              # state arrays of the wrong dtype are not updated in place
        run_set({**p, 'ids': p['ids'].astype(np.int32)})
    with pytest.raises(_lib.Gen6DLibraryError, match='K >= 1'):
        run_set({**p, 'centers': np.zeros((0, 3))})


def test_entry_points_are_declared_and_bound():
    from gen6d_b200 import _lib
    for n in ('g6d_instances_associate_objects', 'g6d_instances_associate_objects_host'):
        assert n in _lib.header_symbols() and n in _lib._SIGNATURES, n


def test_bench_dry_run():
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parents[1]
    out = subprocess.run([sys.executable, str(root / 'tools' / 'objects_instance_track_bench.py'), '--dry-run'], cwd=root,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'dry run' in out.stdout
