"""Tracking an object set (ObjectSet.tracker, gen6d_b200/track.py ObjectTracker) on the H100: the object-indexed glue and
smoothing kernels against their host twins and the per-object launches, one object against est.tracker() bit for bit,
three objects against three single-object trackers, one graph and one read per step with launches independent of K,
free running, isolation, and the errors."""
import os

import numpy as np
import pytest
import torch

from golden import track_cases

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))
SEEDS = {'a': 7, 'b': 8, 'c': 11}
KEYS = ('det_position', 'det_scale_r2q', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores')


@pytest.fixture(scope='module')
def dbs():
    from gen6d_b200.synthetic import synthetic_database
    return {n: synthetic_database(seed=s) for n, s in SEEDS.items()}


@pytest.fixture(scope='module')
def est(dbs):
    from gen6d_b200.synthetic import build_estimator
    e = build_estimator(dbs['a'])[0]
    e.cfg['device_glue'] = True
    return e


@pytest.fixture(scope='module')
def single():
    """A second estimator, rebuilt on each object in turn: the single-object trackers of the comparisons."""
    from gen6d_b200.synthetic import build_estimator
    e = build_estimator()[0]
    e.cfg['device_glue'] = True
    return e


@pytest.fixture(scope='module')
def video(dbs):
    K = TG['track.K']
    return [dbs['a'].render(p, K) for p in TG['track.gt_poses']], K


@pytest.fixture(scope='module')
def objs3(est, dbs):
    objs = est.object_set()
    for n, db in dbs.items():
        objs.add(n, db)
    return objs


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------ 1. kernels
@pytest.mark.parametrize('f32', [0, 1])
def test_glue_kernels_equal_host_twin_and_per_object_launches(objs3, f32):
    from gen6d_b200 import glue, ops
    obs = list(objs3._objects.values())
    K, S, R = len(obs), 2, obs[0].tables['tables']['ref_num']
    views = [ob.tables['views'] for ob in obs]
    tables = [ob.tables['tables'] for ob in obs]
    rng = np.random.RandomState(3 + f32)
    frames = torch.zeros(S, 48, 64, 3, dtype=torch.uint8, device='cuda')
    Ks = np.stack([TG['track.K'] * (1 + 0.01 * s) for s in range(S)], 0)
    Ks[:, 2, 2] = 1
    cams = glue.cameras(Ks)
    poses = []
    for ob, tb in zip(obs, tables):                              # database poses, slightly perturbed
        for i in rng.randint(0, len(tb['ids']), S):
            p = np.asarray(ob.ref.database.get_pose(tb['ids'][i]), np.float64).copy()
            p[:, 3] += rng.randn(3) * 0.02
            poses.append(p)
    poses = np.stack(poses, 0)
    if f32:
        poses = poses.astype(np.float32).astype(np.float64)
    cams_d, poses_d = _dev(cams), _dev(poses.reshape(K * S, 12))
    got = ops.glue_refine_problems_objects(views, R, cams_d, frames, poses_d, f32)
    net = (rng.randn(K * S, 7) * 0.05).astype(np.float32)
    net[:, 0] += 1
    got_poses = ops.glue_apply_refinements_objects(views, got[2], got[1], got[3], _dev(net))
    torch.cuda.synchronize()
    # per-object launches on the slices: bit for bit
    for o in range(K):
        r = slice(o * S, (o + 1) * S)
        want = ops.glue_refine_problems(views[o], R, cams_d, frames, poses_d[r], f32)
        for name, g, w in zip(('jobs', 'que_K', 'que_pose', 'rect', 'ref_Ks', 'ref_poses', 'ref_rows'), got, want):
            g = g.reshape(K * S, -1)[r] if name == 'jobs' else g[r]
            assert torch.equal(g.reshape(-1).view(torch.uint8), w.reshape(-1).view(torch.uint8)), (o, name)
        want_poses = ops.glue_apply_refinements(views[o], want[2], want[1], want[3], _dev(net[r]))
        assert torch.equal(got_poses[r], want_poses), o
    # the host twin: the same code on the CPU
    sources = []
    for ob in obs:
        vd = ob.tables['keep'][1]
        sources.append((vd['src'].cpu().numpy().view(np.uint64), vd['rows'].cpu().numpy(), vd['cols'].cpu().numpy()))
    host = glue.host_refine_problems_objects(tables, cams, poses, f32, 48, 64, frame_ptr=frames.data_ptr(), sources=sources)
    host_poses = glue.host_apply_refinements_objects(tables, host, net)
    jobs = np.frombuffer(got[0].cpu().numpy().tobytes(), glue.JOB)
    worst = 0.0
    for k in ('src', 'rows', 'cols'):
        np.testing.assert_array_equal(jobs[k], host['jobs'][k], err_msg=k)
    np.testing.assert_array_equal(got[6].cpu().numpy(), host['ref_rows'])
    pairs = [(jobs['M'], host['jobs']['M'])] + [(g.cpu().numpy(), host[k]) for g, k in
                                                zip(got[1:6], ('que_K', 'que_pose', 'pose_rect', 'ref_Ks', 'ref_poses'))]
    pairs.append((got_poses.cpu().numpy().reshape(K * S, 3, 4), host_poses))
    bitwise = True
    for g, h in pairs:
        bitwise &= g.tobytes() == h.tobytes()
        worst = max(worst, float(np.abs(g.astype(np.float64) - h).max() / max(np.abs(h).max(), 1e-30)))
    print('object glue, device vs host twin: bit-identical', bitwise, 'max relative difference', worst)
    assert worst <= 1e-6                      # device vs glibc trigonometry, then float32 rounding


@pytest.mark.parametrize('S', [1, 4])
def test_smoothing_kernel_equals_host_twin_and_per_object_launches(S):
    from gen6d_b200 import ops, track as T
    K, num, L = 3, 5, 7
    cases = [[track_cases.smoothing_case(seed=900 + 10 * o + s, L=L) for s in range(S)] for o in range(K)]
    bboxes = np.stack([T.bbox_from_points(cases[o][0]['pts']) for o in range(K)], 0)
    Ks = np.stack([cases[0][s]['K'] for s in range(S)], 0).reshape(S, 9).astype(np.float64)
    w = T.smoothing_weights(num, 2.5)
    ring, count = np.zeros((K * S, num, 8, 2), np.float32), np.zeros(K * S, np.int32)
    ring_d, count_d, bb_d, Ks_d, w_d = _dev(ring), _dev(count), _dev(bboxes), _dev(Ks), _dev(w)
    rings_o = [_dev(np.zeros((S, num, 8, 2), np.float32)) for _ in range(K)]
    counts_o = [_dev(np.zeros(S, np.int32)) for _ in range(K)]
    worst = 0.0
    for k in range(L):
        poses = np.stack([cases[o][s]['poses'][k] for o in range(K) for s in range(S)], 0).astype(np.float64).reshape(K * S, 12)
        sm_d, avg_d = ops.track_smooth_objects(_dev(poses), True, bb_d, Ks_d, ring_d, count_d, w_d)
        sm_h, avg_h = T.host_smooth_objects(poses, True, bboxes, Ks, ring, count, w)
        np.testing.assert_array_equal(ring_d.cpu().numpy(), ring)
        np.testing.assert_array_equal(count_d.cpu().numpy(), count)
        np.testing.assert_array_equal(avg_d.cpu().numpy(), avg_h)
        sm = sm_d.cpu().numpy().reshape(K * S, 3, 4)
        worst = max(worst, float((np.abs(sm - sm_h).reshape(K * S, -1).max(1) / np.abs(sm_h).reshape(K * S, -1).max(1)).max()))
        for o in range(K):
            r = slice(o * S, (o + 1) * S)
            sm_o, avg_o = ops.track_smooth(_dev(poses[r]), True, bb_d[o], Ks_d, rings_o[o], counts_o[o], w_d)
            assert torch.equal(sm_d[r], sm_o) and torch.equal(avg_d[r], avg_o), (k, o)
            assert torch.equal(ring_d[r], rings_o[o]) and torch.equal(count_d[r], counts_o[o]), (k, o)
    print('object smoothing, device vs host twin, max relative |dpose|', worst)
    assert worst <= 1e-9


# ------------------------------------------------------------------------------------------ 2. one object
def _steps(trk, frames, K, name=None):
    out = []
    for f in frames:
        r = trk.step([f], [K])
        out.append(r[name] if name is not None else r)
    return out


def test_one_object_equals_est_tracker(est, dbs, video):
    frames, K = video
    objs = est.object_set()
    objs.add('a', dbs['a'])
    got = _steps(objs.tracker(), frames, K, 'a')
    want = _steps(est.tracker(), frames, K)
    for t, ((p, sm, inter), (wp, wsm, winter)) in enumerate(zip(got, want)):
        assert p.dtype == wp.dtype and p.tobytes() == wp.tobytes(), t
        assert sm.dtype == wsm.dtype and sm.tobytes() == wsm.tobytes(), t
        assert set(winter) <= set(inter), (t, sorted(set(winter) - set(inter)))
        for k in winter:
            if k == 'refine_poses':
                assert len(inter[k]) == len(winter[k]), t
                for x, y in zip(inter[k], winter[k]):
                    assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), (t, k)
            else:
                assert inter[k].dtype == winter[k].dtype and inter[k].shape == winter[k].shape, (t, k)
                assert inter[k].tobytes() == winter[k].tobytes(), (t, k)
        if t == 0:
            assert 'det_score' in inter and inter['det_score'].shape == (1,)
            assert len(inter['refine_poses']) == est.cfg['refine_iter'] + 1
        else:
            assert len(inter['refine_poses']) == 2


# ------------------------------------------------------------------------------------------ 3. three objects
def _pose_dev(got, want):
    return float(np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64)).max())


def test_three_objects_equal_three_trackers(objs3, single, dbs, video):
    from test_objects_gpu import _assert_matches_single
    from gen6d_b200 import track as T
    frames, K = video
    S = 2
    trk = objs3.tracker(num_sequences=S)
    starts = {n: TG['track.raw_poses'][0:S] for n in objs3.names}
    trk.start(starts)
    many = trk.step(frames[1:1 + S], [K] * S)
    trk.reset()
    first = trk.step(frames[0:S], [K] * S)
    more = [trk.step(frames[t:t + S], [K] * S) for t in (2, 4)]
    for n, db in dbs.items():
        single.build(db, 'all')
        one = single.tracker(num_sequences=S)
        one.start(starts[n])
        p1, _, _ = one.step(frames[1:1 + S], [K] * S)
        d = _pose_dev(many[n][0], p1)
        print(n, 'teacher-forced step, 3-object set vs single-object tracker, max |dpose|', d)
        assert d <= 2e-4, (n, d)
        # the full first step: the set's prediction against a single-object predict_batch
        wp, winter = single.predict_batch(frames[0:S], [K] * S)
        _assert_matches_single((first[n][0], first[n][2]), (wp, winter), n)
        # each object's smoothing is host_smooth of its own raw poses (box of its own database)
        ring, count = np.zeros((S, 5, 8, 2), np.float32), np.zeros(S, np.int32)
        box, w = T.object_bbox(db), T.smoothing_weights(5, 2.5)
        worst = 0.0
        for step in [first] + more:
            raw, sm, _ = step[n]
            s_h, _ = T.host_smooth(raw, True, box, np.stack([K] * S, 0), ring, count, w)
            worst = max(worst, float((np.abs(s_h - sm).reshape(S, -1).max(1) / np.abs(s_h).reshape(S, -1).max(1)).max()))
        assert worst <= 1e-12, (n, worst)


# ------------------------------------------------------------------------------------------ 4. one graph, one read
def test_one_graph_one_read_and_launches_independent_of_K(est, objs3, single, dbs, video, monkeypatch):
    from gen6d_b200 import glue, ops
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    frames, K = video
    trk = objs3.tracker()
    trk.step(frames[:1], [K])
    trk.step(frames[1:2], [K])
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    trk.step(frames[2:3], [K])
    stage = [s for key, s in trk.stages.stages.items() if key[0].startswith('track_refine')]
    assert len(stage) == 1 and REPLAYED_KERNELS[0] - k0 == stage[0].kernels      # one replay ...
    assert IO_BYTES['d2h'] - d0 == stage[0].static_out[0].numel()                 # ... and one read
    set_kernels = stage[0].kernels
    # the object-indexed wrappers: 2 * refine_iter + 1 calls per step function, for one object and for three
    objs1 = est.object_set()
    objs1.add('a', dbs['a'])
    names = ('glue_refine_problems_objects', 'glue_apply_refinements_objects', 'track_smooth_objects')
    for objs in (objs1, objs3):
        calls = []
        for nm in names:
            orig = getattr(ops, nm)
            monkeypatch.setattr(ops, nm, lambda *a, _o=orig, _n=nm, **k: (calls.append(_n), _o(*a, **k))[1])
        t = objs.tracker(refine_iter=2)
        t.start({n: TG['track.raw_poses'][0:1] for n in objs.names})
        with torch.no_grad():
            fn = t._refine_fn(False)
            fn(est.detector.upload_frame([frames[1]]), est.detector._to_dev(glue.cameras(np.stack([K], 0))), t._prev, t._ring, t._count)
        torch.cuda.synchronize()
        assert len(calls) == 2 * 2 + 1, (len(objs), calls)
        monkeypatch.undo()
    # fewer kernels than three single-object refine-step graphs
    total = 0
    for n, db in dbs.items():
        single.build(db, 'all')
        one = single.tracker()
        one.step(frames[:1], [K])
        one.step(frames[1:2], [K])
        total += [s for key, s in one.stages.stages.items() if key[0].startswith('track_refine')][0].kernels
    print('3-object refine-step graph kernels', set_kernels, 'vs three single-object graphs', total)
    assert set_kernels < total


# ------------------------------------------------------------------------------------------ 5. free running, isolation
def test_free_running_and_isolation(est, objs3, video):
    frames, K = video
    imgs, Ks = frames[:3], [K] * 3
    before_set = objs3.predict(imgs, Ks)
    before_est = est.predict_batch(imgs, Ks)
    before_trk = _steps(est.tracker(), frames[:3], K)
    trk = objs3.tracker()
    a = _steps(trk, frames, K)
    trk.reset()
    b = _steps(trk, frames, K)
    for t, (x, y) in enumerate(zip(a, b)):
        for n in objs3.names:
            assert np.isfinite(x[n][0]).all() and np.isfinite(x[n][1]).all(), (t, n)
            np.testing.assert_array_equal(x[n][0], y[n][0], err_msg=f'{t} {n}')
            np.testing.assert_array_equal(x[n][1], y[n][1], err_msg=f'{t} {n}')
    after_set = objs3.predict(imgs, Ks)
    after_est = est.predict_batch(imgs, Ks)
    after_trk = _steps(est.tracker(), frames[:3], K)
    for n in before_set:
        np.testing.assert_array_equal(before_set[n][0], after_set[n][0], err_msg=n)
        for k in KEYS + ('det_score',):
            np.testing.assert_array_equal(before_set[n][1][k], after_set[n][1][k], err_msg=f'{n} {k}')
    np.testing.assert_array_equal(before_est[0], after_est[0])
    for k in KEYS:
        np.testing.assert_array_equal(before_est[1][k], after_est[1][k], err_msg=k)
    for x, y in zip(before_trk, after_trk):
        np.testing.assert_array_equal(x[0], y[0])
        np.testing.assert_array_equal(x[1], y[1])


# ------------------------------------------------------------------------------------------ 6. errors and staleness
def test_errors_and_staleness(single, dbs, video):
    frames, K = video
    objs = single.object_set()
    objs.add('a', dbs['a'])
    objs.add('b', dbs['b'])
    for kw in ({'num_sequences': 0}, {'refine_iter': 0}, {'smooth_num': 0}, {'smooth_std': 0.0},
               {'bboxes': {'a': np.zeros((8, 3), np.float32)}}, {'bboxes': {'x': TG['track.bbox']}}):
        with pytest.raises(ValueError):
            objs.tracker(**kw)
    trk = objs.tracker(num_sequences=2)
    with pytest.raises(ValueError):
        trk.step(frames[:1], [K])                                   # one frame for two sequences
    with pytest.raises(ValueError):
        trk.step(frames[:2], [K])                                   # one K for two sequences
    with pytest.raises(ValueError):
        trk.start({'a': TG['track.raw_poses'][0:2]})                # 'b' missing
    with pytest.raises(ValueError):
        trk.start({'a': TG['track.raw_poses'][0:2].astype(np.float32), 'b': TG['track.raw_poses'][0:2].astype(np.float64)})
    with pytest.raises(ValueError):
        trk.start({'a': TG['track.raw_poses'][0:1], 'b': TG['track.raw_poses'][0:1]})
    refine_iter = single.cfg['refine_iter']
    trk.step(frames[:2], [K, K])
    trk.step(frames[1:3], [K, K])
    assert single.cfg['refine_iter'] == refine_iter                 # tracking never rewrites the estimator's cfg
    objs.add('c', dbs['c'])
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(frames[:2], [K, K])
    trk = objs.tracker()
    objs.remove('c')
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(frames[:1], [K])
    trk = objs.tracker()
    trk.step(frames[:1], [K])
    single.selector.load_state_dict(single.selector.state_dict())
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(frames[1:2], [K])
