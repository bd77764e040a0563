"""Multi-instance tracking of an object set (ObjectSet.instance_tracker, gen6d_b200/instance_track.py
ObjectInstanceTracker) on the H100: the object-indexed association kernel against its host twin, one object against
est.instance_tracker() bit for bit, M = 1 against objs.tracker() bit for bit, the first step against
objs.predict_instances, two objects against two single-object instance trackers, re-detection, reset of one sequence,
one replay and one read per step over two graphs, and the errors."""
import numpy as np
import pytest
import torch

from tests.test_instance_track_gpu import DET_KEYS, _pose_bound

pytestmark = pytest.mark.gpu
SEEDS = {'a': 7, 'b': 8}


@pytest.fixture(scope='module')
def dbs():
    from gen6d_b200.synthetic import synthetic_database
    return {n: synthetic_database(seed=s) for n, s in SEEDS.items()}


@pytest.fixture(scope='module')
def est(dbs):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(dbs['a'])[0]


@pytest.fixture(scope='module')
def single():
    """A second estimator, rebuilt on each object in turn: the single-object instance trackers of the comparisons."""
    from gen6d_b200.synthetic import build_estimator
    return build_estimator()[0]


@pytest.fixture(scope='module')
def objs2(est, dbs):
    objs = est.object_set()
    for n, db in dbs.items():
        objs.add(n, db)
    return objs


@pytest.fixture(scope='module')
def videos(dbs):
    """Three sequences of 8 frames: two copies of object a and one of object b, at different offsets."""
    from gen6d_b200.synthetic import instance_video
    return [instance_video([(dbs['a'], 2), (dbs['b'], 1)], 8, shift) for shift in (0.0, 6.0, -6.0)]


def _frames(videos, t, S):
    return [videos[s][0][t] for s in range(S)], [videos[s][1] for s in range(S)]


def _same(x, y, msg):
    x, y = np.asarray(x), np.asarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, (msg, x.dtype, y.dtype, x.shape, y.shape)
    assert x.tobytes() == y.tobytes(), msg


def _same_step(got, want, t):
    """(poses, smoothed, ids, inter) of two trackers, bit for bit in every output and inter key."""
    for i, nm in enumerate(('poses', 'smoothed', 'ids')):
        _same(got[i], want[i], f'{t} {nm}')
    assert set(got[3]) == set(want[3]), (t, sorted(set(got[3]) ^ set(want[3])))
    for k, w in want[3].items():
        if k == 'refine_poses':
            assert len(got[3][k]) == len(w), t
            for j, (x, y) in enumerate(zip(got[3][k], w)):
                _same(x, y, f'{t} {k}[{j}]')
        elif k == 'dropped':
            assert got[3][k] == w, t
        else:
            _same(got[3][k], w, f'{t} {k}')


# ------------------------------------------------------------------------------------------ 1. the kernel and its host twin
def test_associate_kernel_equals_host_twin():
    from gen6d_b200 import ops
    from gen6d_b200.instance_track import host_associate_objects
    from tests.test_instance_track_cpu import OUTS, STATE
    from tests.test_objects_instance_track_cpu import ARGS, make_set_problem
    rng = np.random.RandomState(98)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    big = 0
    for trial in range(300):
        K = int(rng.choice([1, 2, 3, 5]))
        p, K, S, M = make_set_problem(rng, K, S=int(rng.choice([1, 3, 10, 60, 300])))
        big += K * S > 256
        h = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
        want = dict(zip(OUTS, host_associate_objects(*[h[k] for k in ARGS], *[h[k] for k in STATE])))
        d = {k: dev(p[k]) for k in STATE}
        got = dict(zip(OUTS, ops.instances_associate_objects(dev(p['det']), dev(p['valid']), dev(p['init']), dev(p['cams']),
                                                             dev(p['centers']), p['res'], p['gate'], p['max_misses'], p['F'], p['r'],
                                                             dev(p['prev']), *[d[k] for k in STATE])))
        for k in OUTS:
            np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=f'{trial} {k}')
        for k in STATE:
            np.testing.assert_array_equal(d[k].cpu().numpy(), h[k], err_msg=f'{trial} {k}')
    assert big > 20, big


# ------------------------------------------------------------------------------------------ 2. one object is est.instance_tracker
def test_one_object_equals_est_instance_tracker(est, dbs, videos):
    S, M = 2, 2
    objs = est.object_set()
    objs.add('a', dbs['a'])
    got_trk = objs.instance_tracker(num_sequences=S, max_instances=M, redetect_every=2)
    want_trk = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=2)
    for t in range(8):
        imgs, Ks = _frames(videos, t, S)
        got = got_trk.step(imgs, Ks)
        assert list(got) == ['a']
        _same_step(got['a'], want_trk.step(imgs, Ks), t)


# ------------------------------------------------------------------------------------------ 3. M = 1 is objs.tracker()
def test_one_instance_equals_object_tracker(objs2, videos):
    S = 2
    trk, itrk = objs2.tracker(num_sequences=S), objs2.instance_tracker(num_sequences=S, max_instances=1)
    for t in range(6):
        imgs, Ks = _frames(videos, t, S)
        want, got = trk.step(imgs, Ks), itrk.step(imgs, Ks)
        for o, n in enumerate(objs2.names):
            p, sm, inter = want[n]
            ip, ism, ids, iinter = got[n]
            _same(ip[:, 0], p, f'{t} {n} poses')
            _same(ism[:, 0], sm, f'{t} {n} smoothed')
            assert len(iinter['refine_poses']) == len(inter['refine_poses']), t
            for x, y in zip(iinter['refine_poses'], inter['refine_poses']):
                _same(x[:, 0], y, f'{t} {n} refine_poses')
            for k in ('bbox_pts', 'smoothed_pts'):
                _same(iinter[k][:, 0], inter[k], f'{t} {n} {k}')
            np.testing.assert_array_equal(ids[:, 0], o * S + np.arange(S))
            if t == 0:
                for k in DET_KEYS:
                    _same(iinter[k][:, 0], inter[k], f'{n} {k}')


# ------------------------------------------------------------------------------------------ 4. the first step
def test_first_step_equals_predict_instances(objs2, videos):
    S, M = 3, 3
    imgs, Ks = _frames(videos, 0, S)
    want = objs2.predict_instances(imgs, Ks, max_instances=M)
    got = objs2.instance_tracker(num_sequences=S, max_instances=M).step(imgs, Ks)
    base = 0
    for n in objs2.names:
        want_p, w = want[n]
        p, sm, ids, inter = got[n]
        valid = w['instance_valid']
        print(n, 'instance counts', w['instance_count'])
        assert valid[:, 0].all()
        np.testing.assert_array_equal(inter['instance_valid'], valid)
        _same(p[valid], want_p[valid], n)
        assert np.isnan(p[~valid]).all() and np.isnan(sm[~valid]).all() and np.isnan(inter['bbox_pts'][~valid]).all()
        assert len(inter['refine_poses']) == len(w['refine_poses'])
        for x, y in zip(inter['refine_poses'], w['refine_poses']):
            _same(x[valid], y[valid], n)
        for k in DET_KEYS + ('instance_count',):
            _same(inter[k], w[k], f'{n} {k}')
        np.testing.assert_array_equal(inter['det_slot'], np.where(valid, np.arange(M)[None], -1))
        np.testing.assert_array_equal(inter['spawned'], valid)
        first = base + np.concatenate([[0], np.cumsum(w['instance_count'])[:-1]])       # (object, sequence, detection) order
        np.testing.assert_array_equal(ids, np.where(valid, first[:, None] + np.arange(M)[None], -1))
        base += int(w['instance_count'].sum())


# ------------------------------------------------------------------------------------------ 5. two objects vs single trackers
def test_two_objects_equal_single_object_trackers(objs2, single, dbs, videos):
    S, M = 2, 2
    imgs, Ks = _frames(videos, 0, S)
    got = objs2.instance_tracker(num_sequences=S, max_instances=M, gate=1e6).step(imgs, Ks)
    offset = 0
    for n, db in dbs.items():
        single.build(db, 'all')
        want = single.instance_tracker(num_sequences=S, max_instances=M, gate=1e6).step(imgs, Ks)
        p, sm, ids, inter = got[n]
        wp, wsm, wids, w = want
        # the set's shared correlation GEMM sums in another order than a single-object detector, so the boxes and scores agree to a few ulps
        for k in ('det_position', 'det_scale_r2q', 'det_score'):
            np.testing.assert_allclose(inter[k], w[k], rtol=1e-5, atol=1e-5, err_msg=f'{n} {k}')
        np.testing.assert_array_equal(inter['sel_ref_idx'], w['sel_ref_idx'], err_msg=n)
        crop_dev = np.abs(inter['det_que_img'].astype(np.int32) - w['det_que_img'].astype(np.int32))
        print(n, 'crops: pixels that differ', int((crop_dev > 0).sum()), 'max', int(crop_dev.max()), 'selected views',
              inter['sel_ref_idx'].tolist(), w['sel_ref_idx'].tolist())
        assert (crop_dev > 0).mean() < 1e-3, n
        for k in ('instance_valid', 'instance_count', 'det_slot', 'spawned'):
            np.testing.assert_array_equal(inter[k], w[k], err_msg=f'{n} {k}')
        # a crop cut from a box an ulp away can differ by one level in a few pixels; its scores then move by up to ~1e-2
        same_crop = (crop_dev.reshape(S, M, -1) == 0).all(-1)
        np.testing.assert_allclose(inter['sel_scores'][same_crop], w['sel_scores'][same_crop], atol=3e-4, err_msg=n)
        np.testing.assert_allclose(inter['sel_scores'], w['sel_scores'], atol=1e-2, err_msg=n)
        np.testing.assert_array_equal(ids >= 0, wids >= 0)
        np.testing.assert_array_equal(ids[ids >= 0], wids[wids >= 0] + offset)
        offset += int((wids >= 0).sum())
        live = ids >= 0
        rows = live & same_crop
        _pose_bound([r[rows] for r in inter['refine_poses']], [r[rows] for r in w['refine_poses']], f'object {n} vs single tracker')
        other = live & ~same_crop                                      # a crop one level off in a few pixels: a looser bar
        if other.any():
            dev = [float(np.abs(np.asarray(x[other], np.float64) - np.asarray(y[other], np.float64)).max())
                   for x, y in zip(inter['refine_poses'], w['refine_poses'])]
            print(n, 'rows with a differing crop: max |dpose| per iteration', dev)
            assert dev[0] < 1e-3 and max(dev) < 0.2, (n, dev)


# ------------------------------------------------------------------------------------------ 6. re-detection
def test_redetection_keeps_or_replaces_ids(objs2, videos):
    S, M = 2, 2
    trk = objs2.instance_tracker(num_sequences=S, max_instances=M, gate=1e6, redetect_every=2)
    first = trk.step(*_frames(videos, 0, S))
    trk.step(*_frames(videos, 1, S))
    again = trk.step(*_frames(videos, 2, S))                          # a re-detection step
    for n in objs2.names:
        ids0, ids1, inter = first[n][2], again[n][2], again[n][3]
        assert 'det_slot' in inter and inter['dropped'] == []
        np.testing.assert_array_equal(ids1[ids0 >= 0], ids0[ids0 >= 0])

    tiny = objs2.instance_tracker(num_sequences=S, max_instances=M, gate=1e-12, max_misses=0, redetect_every=1)
    a = tiny.step(*_frames(videos, 0, S))
    b = tiny.step(*_frames(videos, 1, S))
    prev_max = max(int(a[n][2].max()) for n in objs2.names)
    for n in objs2.names:
        ids_a, ids_b, inter = a[n][2], b[n][2], b[n][3]
        assert inter['dropped'] == sorted(ids_a[ids_a >= 0].tolist())
        np.testing.assert_array_equal(inter['spawned'], inter['instance_valid'])
        assert ((ids_b >= 0) == inter['instance_valid']).all()
        assert (ids_b[ids_b >= 0] > prev_max).all()                   # fresh, and after every earlier object's new ids
        prev_max = max(prev_max, int(ids_b.max()))


# ------------------------------------------------------------------------------------------ 7. reset of one sequence
def test_reset_one_sequence(objs2, videos):
    S, M = 3, 2
    trk = objs2.instance_tracker(num_sequences=S, max_instances=M, gate=1e6)
    ids0 = {n: v[2] for n, v in trk.step(*_frames(videos, 0, S)).items()}
    ids1 = {n: v[2] for n, v in trk.step(*_frames(videos, 1, S)).items()}
    for n in objs2.names:
        np.testing.assert_array_equal(ids1[n], ids0[n])
    trk.reset([1])
    out = trk.step(*_frames(videos, 2, S))                            # re-detects every sequence
    top = max(int(v.max()) for v in ids0.values())
    for n in objs2.names:
        ids2, inter = out[n][2], out[n][3]
        assert 'det_slot' in inter
        for s in (0, 2):
            np.testing.assert_array_equal(ids2[s][ids0[n][s] >= 0], ids0[n][s][ids0[n][s] >= 0])
        assert (ids2[1][ids2[1] >= 0] > top).all() and inter['spawned'][1].any() and not inter['spawned'][[0, 2]].any(), n


# ------------------------------------------------------------------------------------------ 8. one replay, one read, two graphs
def test_one_graph_and_one_read_per_step(est, dbs, objs2, videos):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    S = 2
    objs1 = est.object_set()
    objs1.add('a', dbs['a'])
    refine_kernels = {}
    for objs, M in ((objs1, 4), (objs2, 2)):                          # M*K*S = 8 rows each: one refiner batch size
        trk = objs.instance_tracker(num_sequences=S, max_instances=M, redetect_every=2)
        kinds = []
        for t in range(4):
            k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
            out = trk.step(*_frames(videos, t, S))
            kind = 'detect' if 'det_slot' in out['a'][3] else 'refine'
            kinds.append(kind)
            stage = next(s for key, s in trk.stages.stages.items() if key[0] == kind)
            assert REPLAYED_KERNELS[0] - k0 == stage.kernels, t
            assert IO_BYTES['d2h'] - d0 == stage.static_out[0].numel(), t
        assert kinds == ['detect', 'refine'] * 2
        assert len(trk.stages.stages) == 2
        kernels = {key[0]: s.kernels for key, s in trk.stages.stages.items()}
        print(len(objs), 'objects x', M, 'slots: graph kernels', kernels)
        refine_kernels[len(objs)] = kernels['refine']
    assert refine_kernels[2] == refine_kernels[1]                     # M*K <= 16: one glue launch per step function


# ------------------------------------------------------------------------------------------ 9. errors and staleness
def test_errors_and_staleness(single, dbs, videos):
    objs = single.object_set()
    objs.add('a', dbs['a'])
    objs.add('b', dbs['b'])
    for kw in (dict(max_instances=0), dict(max_instances=17), dict(nms_iou=1.5), dict(peak_radius=4), dict(min_score=float('nan')),
               dict(gate=0.0), dict(gate=float('inf')), dict(max_misses=-1), dict(redetect_every=0), dict(refine_iter=0),
               dict(num_sequences=0), dict(smooth_num=0), dict(smooth_std=0.0),
               dict(bboxes={'a': np.zeros((8, 3), np.float32)}), dict(bboxes={'x': np.ones((8, 3), np.float32)})):
        with pytest.raises(ValueError):
            objs.instance_tracker(**kw)
    with pytest.raises(ValueError, match='empty'):
        single.object_set().instance_tracker()
    trk = objs.instance_tracker(num_sequences=2, max_instances=2)
    with pytest.raises(ValueError):
        trk.step(*_frames(videos, 0, 1))
    with pytest.raises(ValueError):
        trk.reset([2])
    trk.step(*_frames(videos, 0, 2))
    objs.add('c', dbs['a'])
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(*_frames(videos, 1, 2))
    trk = objs.instance_tracker(num_sequences=2, max_instances=2)
    objs.remove('c')
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(*_frames(videos, 1, 2))
    trk = objs.instance_tracker(num_sequences=2, max_instances=2)
    trk.step(*_frames(videos, 0, 2))
    single.selector.load_state_dict(single.selector.state_dict())     # new weights (same values): the tracker goes stale
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(*_frames(videos, 1, 2))
