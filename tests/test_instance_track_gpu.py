"""Multi-instance tracking (Gen6DEstimator.instance_tracker) on the H100: M = 1 against est.tracker() bit for bit, the first
step against predict_instances bit for bit, the association kernel against its host twin, re-detection with a wide and a
tiny gate, reset of one sequence, one replay and one read per step over two graphs, and the errors."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENS = np.load(os.path.join(HERE, 'golden', 'sens_golden.npz'))
DET_KEYS = ('det_position', 'det_scale_r2q', 'det_score', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores')


@pytest.fixture(scope='module')
def db():
    from gen6d_b200.synthetic import synthetic_database
    return synthetic_database(seed=7)


@pytest.fixture(scope='module')
def est(db):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(db)[0]


def two_copy_video(db, T, shift=0.0):
    """T frames of two copies of the object translating across the frame (test_instances_gpu.py's compositing)."""
    i = db.get_img_ids()[3]
    pose, K = db.poses[i].copy(), db.get_K(i)
    frames = []
    for t in range(T):
        dx = shift + 4.0 * t
        a, b = pose.copy(), pose.copy()
        a[0, 3] += (dx - 120.0) * pose[2, 3] / K[0, 0]
        b[0, 3] += (dx + 220.0) * pose[2, 3] / K[0, 0]
        ia, ib = db.render(a, K), db.render(b, K)
        frames.append(np.where((ib != db._bg).any(-1, keepdims=True), ib, ia))
    return frames, K


@pytest.fixture(scope='module')
def videos(db):
    """Three sequences of 8 frames (the copies at different offsets)."""
    return [two_copy_video(db, 8, shift) for shift in (0.0, 15.0, -10.0)]


def _frames(videos, t, S):
    return [videos[s][0][t] for s in range(S)], [videos[s][1] for s in range(S)]


def _pose_bound(a, b, name):
    """The sensitivity bar of test_instances_gpu.py."""
    a = np.stack([np.asarray(p, np.float64) for p in a])
    b = np.stack([np.asarray(p, np.float64) for p in b])
    dev = np.abs(a - b).reshape(len(a), -1).max(1)
    print(name, 'max |dpose| per iteration', dev)
    assert dev[0] < 1e-4, (name, dev)
    assert (dev[1:] <= np.maximum(2.0 * SENS['gain_R'][1:] * 1e-3, 2e-3)).all(), (name, dev)


# ------------------------------------------------------------------------------------------ 1. M = 1 is the tracker
def test_one_instance_equals_tracker(est, videos):
    S = 2
    trk, itrk = est.tracker(num_sequences=S), est.instance_tracker(num_sequences=S, max_instances=1)
    for t in range(8):
        imgs, Ks = _frames(videos, t, S)
        p, sm, inter = trk.step(imgs, Ks)
        ip, ism, ids, iinter = itrk.step(imgs, Ks)
        assert ip.shape == (S, 1, 3, 4) and ip.dtype == p.dtype and ism.dtype == sm.dtype
        np.testing.assert_array_equal(ip[:, 0], p, err_msg=str(t))
        np.testing.assert_array_equal(ism[:, 0], sm, err_msg=str(t))
        assert len(iinter['refine_poses']) == len(inter['refine_poses']), t
        for x, y in zip(iinter['refine_poses'], inter['refine_poses']):
            assert x.dtype == y.dtype, t
            np.testing.assert_array_equal(x[:, 0], y, err_msg=str(t))
        for k in ('bbox_pts', 'smoothed_pts'):
            assert iinter[k].dtype == inter[k].dtype, k
            np.testing.assert_array_equal(iinter[k][:, 0], inter[k], err_msg=f'{t} {k}')
        np.testing.assert_array_equal(ids, [[0], [1]])
        if t == 0:
            for k in ('det_position', 'det_scale_r2q', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores'):
                np.testing.assert_array_equal(iinter[k][:, 0], inter[k], err_msg=k)
            assert iinter['spawned'].all() and iinter['dropped'] == []
        else:
            assert 'spawned' not in iinter


# ------------------------------------------------------------------------------------------ 2. the first step
def test_first_step_equals_predict_instances(est, videos):
    S, M = 3, 3
    imgs, Ks = _frames(videos, 0, S)
    want_p, want = est.predict_instances(imgs, Ks, max_instances=M)
    p, sm, ids, inter = est.instance_tracker(num_sequences=S, max_instances=M).step(imgs, Ks)
    valid = want['instance_valid']
    assert valid[:, 0].all()
    print('instance counts', want['instance_count'])
    np.testing.assert_array_equal(inter['instance_valid'], valid)
    np.testing.assert_array_equal(p[valid], want_p[valid])
    assert np.isnan(p[~valid]).all() and np.isnan(sm[~valid]).all() and np.isnan(inter['bbox_pts'][~valid]).all()
    assert len(inter['refine_poses']) == len(want['refine_poses'])
    for x, y in zip(inter['refine_poses'], want['refine_poses']):
        assert x.dtype == y.dtype
        np.testing.assert_array_equal(x[valid], y[valid])
    for k in DET_KEYS + ('instance_count',):
        np.testing.assert_array_equal(inter[k], want[k], err_msg=k)
    np.testing.assert_array_equal(inter['det_slot'], np.where(valid, np.arange(M)[None], -1))
    np.testing.assert_array_equal(inter['spawned'], valid)
    first = np.concatenate([[0], np.cumsum(want['instance_count'])[:-1]])
    np.testing.assert_array_equal(ids, np.where(valid, first[:, None] + np.arange(M)[None], -1))


# ------------------------------------------------------------------------------------------ 3. the kernel and its host twin
def test_associate_kernel_equals_host_twin():
    from gen6d_b200 import ops
    from gen6d_b200.instance_track import host_associate
    from tests.test_instance_track_cpu import OUTS, STATE, make_problem
    rng = np.random.RandomState(99)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for trial in range(300):
        p = make_problem(rng, S=int(rng.choice([1, 3, 10, 40, 300])))
        h = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
        args = [h[k] for k in ('det', 'valid', 'init', 'cams', 'center', 'res', 'gate', 'max_misses', 'F', 'r', 'prev')]
        want = dict(zip(OUTS, host_associate(*args, *[h[k] for k in STATE])))
        d = {k: dev(p[k]) for k in STATE}
        got = dict(zip(OUTS, ops.instances_associate(dev(p['det']), dev(p['valid']), dev(p['init']), dev(p['cams']), p['center'],
                                                     p['res'], p['gate'], p['max_misses'], p['F'], p['r'], dev(p['prev']),
                                                     *[d[k] for k in STATE])))
        for k in OUTS:
            np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=f'{trial} {k}')
        for k in STATE:
            np.testing.assert_array_equal(d[k].cpu().numpy(), h[k], err_msg=f'{trial} {k}')


# ------------------------------------------------------------------------------------------ 4. re-detection
def test_redetection_keeps_or_replaces_ids(est, videos):
    S, M, r = 2, 2, 1
    trk = est.instance_tracker(num_sequences=S, max_instances=M, gate=1e6, redetect_every=2)
    imgs, Ks = _frames(videos, 0, S)
    _, _, ids0, i0 = trk.step(imgs, Ks)
    live0 = ids0 >= 0
    assert live0[:, 0].all()
    trk.step(*_frames(videos, 1, S))
    imgs, Ks = _frames(videos, 2, S)
    _, _, ids1, inter = trk.step(imgs, Ks)                            # a re-detection step
    assert 'det_slot' in inter and inter['dropped'] == []
    np.testing.assert_array_equal(ids1[live0], ids0[live0])          # every track matched: every id kept
    cont = live0 & ~inter['spawned']
    assert cont.any()
    rows = np.argwhere(cont)
    with torch.no_grad():
        fr = est.detector.upload_frame([np.asarray(imgs[s]) for s, _ in rows])
        p0 = np.stack([inter['refine_poses'][0][s, m] for s, m in rows]).astype(np.float32)
        _, chain = est._refine_batch_host(fr, [np.asarray(Ks[s]) for s, _ in rows], p0, r)
    got = [np.stack([c[s, m] for s, m in rows]) for c in inter['refine_poses'][:r + 1]]
    _pose_bound(got, chain, 'continuing tracks vs host refinement')

    tiny = est.instance_tracker(num_sequences=S, max_instances=M, gate=1e-12, max_misses=0, redetect_every=1)
    _, _, a, _ = tiny.step(*_frames(videos, 0, S))
    _, _, b, inter = tiny.step(*_frames(videos, 1, S))
    assert inter['dropped'] == sorted(a[a >= 0].tolist())
    np.testing.assert_array_equal(inter['spawned'], inter['instance_valid'])
    assert (b[b >= 0] > a.max()).all() and ((b >= 0) == inter['instance_valid']).all()


# ------------------------------------------------------------------------------------------ 5. reset of one sequence
def test_reset_one_sequence(est, videos):
    S, M = 3, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, gate=1e6)
    _, _, ids0, _ = trk.step(*_frames(videos, 0, S))
    _, _, ids1, _ = trk.step(*_frames(videos, 1, S))
    np.testing.assert_array_equal(ids1, ids0)
    trk.reset([1])
    _, _, ids2, inter = trk.step(*_frames(videos, 2, S))              # re-detects every sequence
    assert 'det_slot' in inter
    for s in (0, 2):
        np.testing.assert_array_equal(ids2[s][ids0[s] >= 0], ids0[s][ids0[s] >= 0])
    assert (ids2[1][ids2[1] >= 0] > ids0.max()).all() and inter['spawned'][1].any() and not inter['spawned'][[0, 2]].any()


# ------------------------------------------------------------------------------------------ 6. one replay, one read, two graphs
def test_one_graph_and_one_read_per_step(est, videos):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    S, M = 2, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=2)
    kinds = []
    for t in range(6):
        k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
        out = trk.step(*_frames(videos, t, S))
        kind = 'detect' if 'det_slot' in out[3] else 'refine'
        kinds.append(kind)
        stage = next(s for key, s in trk.stages.stages.items() if key[0] == kind)
        assert REPLAYED_KERNELS[0] - k0 == stage.kernels, t
        assert IO_BYTES['d2h'] - d0 == stage.static_out[0].numel(), t
    assert kinds == ['detect', 'refine'] * 3
    assert len(trk.stages.stages) == 2
    print('graph kernels', {key[0]: s.kernels for key, s in trk.stages.stages.items()})


# ------------------------------------------------------------------------------------------ 7. errors and staleness
def test_errors_and_staleness(est, db, videos):
    import types
    from gen6d_b200.estimator import Gen6DEstimator
    for kw in (dict(max_instances=0), dict(max_instances=17), dict(nms_iou=1.5), dict(peak_radius=4), dict(min_score=float('nan')),
               dict(gate=0.0), dict(gate=float('inf')), dict(max_misses=-1), dict(redetect_every=0), dict(refine_iter=0),
               dict(num_sequences=0), dict(smooth_num=0), dict(smooth_std=0.0)):
        with pytest.raises(ValueError):
            est.instance_tracker(**kw)
    no_refiner = Gen6DEstimator({}, modules={'detector': est.detector, 'selector': est.selector})
    with pytest.raises(ValueError, match='refiner'):
        no_refiner.instance_tracker()
    comm = est.selector.comm
    try:
        est.selector.comm = types.SimpleNamespace(world=2, capturable=False)
        with pytest.raises(ValueError, match='sharded'):
            est.instance_tracker()
    finally:
        est.selector.comm = comm
    est.cfg['host_warps'] = True
    try:
        with pytest.raises(ValueError, match='host_warps'):
            est.instance_tracker()
    finally:
        est.cfg['host_warps'] = False
    trk = est.instance_tracker(num_sequences=2, max_instances=2)
    with pytest.raises(ValueError):
        trk.step(*_frames(videos, 0, 1))
    with pytest.raises(ValueError):
        trk.reset([2])
    first = trk.step(*_frames(videos, 0, 2))
    est.selector.load_state_dict(est.selector.state_dict())           # new weights (same values): the tracker goes stale
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(*_frames(videos, 1, 2))
    est.build(db, 'all')
    again = est.instance_tracker(num_sequences=2, max_instances=2).step(*_frames(videos, 0, 2))
    np.testing.assert_array_equal(first[0], again[0])
    np.testing.assert_array_equal(first[2], again[2])
