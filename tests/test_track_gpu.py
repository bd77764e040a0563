"""Video tracking on the H100: the smoothing kernel against its host twin and the reference's smoothing, tracking steps
against the unmodified reference's tracking run (track_golden.npz), the captured step graph against the host-sequenced
path, lockstep sequences against single ones, and the tracker's errors."""
import os

import numpy as np
import pytest
import torch

from golden import track_cases

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    return build_estimator()


@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K']
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _pose_dev(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    dR = float(np.abs(got[..., :3] - want[..., :3]).max())
    dt = float((np.abs(got[..., 3] - want[..., 3]).max(-1) / np.linalg.norm(want[..., 3], axis=-1)).max())
    return dR, dt


def _set_glue(e, on):
    was = e.cfg['device_glue']
    e.cfg['device_glue'] = on
    return was


def test_device_kernel_equals_host_twin():
    """512 random histories: the corners and their average bit for bit (same code, no FMA contraction), the PnP poses to
    the device's vs glibc's sin / cos / acos rounding.  Levenberg-Marquardt stops once a step changes the parameters by
    less than FLT_EPSILON relative, so a last-ulp difference can end one sequence's solve one iteration earlier on one
    side: the poses then differ by that last (sub-FLT_EPSILON) step, hence a bound of 1e-9 rather than a few ulp."""
    from gen6d_b200 import ops, track as T
    S, num = 512, 5
    cs = [track_cases.smoothing_case(seed=5000 + s, L=9) for s in range(S)]
    bbox = T.bbox_from_points(cs[0]['pts'])
    Ks = np.stack([c['K'] for c in cs], 0).reshape(S, 9).astype(np.float64)
    w = T.smoothing_weights(num, 2.5)
    ring, count = np.zeros((S, num, 8, 2), np.float32), np.zeros(S, np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ring_d, count_d, bbox_d, Ks_d, w_d = dev(ring), dev(count), dev(bbox), dev(Ks), dev(w)
    worst = 0.0
    for k in range(9):
        poses = np.stack([c['poses'][k] for c in cs], 0)
        sm_h, avg_h = T.host_smooth(poses, True, bbox, Ks, ring, count, w)
        sm_d, avg_d = ops.track_smooth(dev(poses.astype(np.float64).reshape(S, 12)), True, bbox_d, Ks_d, ring_d, count_d, w_d)
        np.testing.assert_array_equal(ring_d.cpu().numpy(), ring)
        np.testing.assert_array_equal(count_d.cpu().numpy(), count)
        np.testing.assert_array_equal(avg_d.cpu().numpy(), avg_h)
        sm_d = sm_d.cpu().numpy().reshape(S, 3, 4)
        rel = float((np.abs(sm_d - sm_h).reshape(S, -1).max(1) / np.abs(sm_h).reshape(S, -1).max(1)).max())
        worst = max(worst, rel)
    print('device vs host smoothing, max relative |dpose|', worst)
    assert worst <= 1e-9


def test_device_smoothing_of_golden_raw_poses():
    from gen6d_b200 import ops, track as T
    num, std = int(TG['track.num']), float(TG['track.std'])
    raw, K, bbox = TG['track.raw_poses'], TG['track.K'], TG['track.bbox']
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ring, count = dev(np.zeros((1, num, 8, 2), np.float32)), dev(np.zeros(1, np.int32))
    w, Kd, bd = dev(T.smoothing_weights(num, std)), dev(K.astype(np.float64).reshape(1, 9)), dev(bbox)
    worst = (0.0, 0.0)
    for k in range(len(raw)):
        sm, avg = ops.track_smooth(dev(raw[k].astype(np.float64).reshape(1, 12)), True, bd, Kd, ring, count, w)
        np.testing.assert_allclose(avg.cpu().numpy()[0], TG['track.avg'][k], rtol=1e-6)
        d = _pose_dev(sm.cpu().numpy().reshape(3, 4), TG['track.smoothed'][k])
        worst = (max(worst[0], d[0]), max(worst[1], d[1]))
    print('golden raw poses smoothed on the device: max |dR|', worst[0], 'relative |dt|', worst[1])
    assert worst[0] <= 1e-7 and worst[1] <= 1e-7


def _teacher_forced(e, frames, K, device_glue, S=1, ts=range(1, 8)):
    was = _set_glue(e, device_glue)
    try:
        trk = e.tracker(num_sequences=S)
        out = []
        for t in ts:
            trk.start(TG['track.raw_poses'][t - 1][None])
            poses, _, inter = trk.step([frames[t]], [K])
            assert len(inter['refine_poses']) == 2
            out.append(poses[0])
        return np.stack(out, 0)
    finally:
        e.cfg['device_glue'] = was


def test_teacher_forced_steps_match_reference(est, video):
    """From the reference's own raw pose of frame t-1, one tracked step on frame t reproduces its raw pose of frame t
    (the bar of test_tracking_refinement_matches_reference)."""
    e, _ = est
    frames, K = video
    got = _teacher_forced(e, frames, K, True)
    want = TG['track.raw_poses'][1:]
    for t in range(len(got)):
        dR, dt = _pose_dev(got[t], want[t])
        print(f'frame {t + 1}: max |dR| {dR:.3e} relative |dt| {dt:.3e}')
    np.testing.assert_allclose(got[:, :, :3], want[:, :, :3], atol=1e-2)
    assert _pose_dev(got, want)[1] < 1e-2


def test_teacher_forced_graph_equals_host_path(est, video):
    e, _ = est
    frames, K = video
    dev = _teacher_forced(e, frames, K, True)
    host = _teacher_forced(e, frames, K, False)
    d = float(np.abs(dev.astype(np.float64) - host).max())
    print('teacher-forced step, device graph vs host path, max |dpose|', d)
    assert d <= 2e-4


def test_first_step_equals_predict_batch(est, video):
    """The first step is predict_batch's captured device-glue graph with the smoothing kernel appended."""
    e, _ = est
    frames, K = video
    was = _set_glue(e, True)
    try:
        want_poses, want = e.predict_batch(frames[:2], [K, K])
        trk = e.tracker(num_sequences=2)
        poses, smoothed, inter = trk.step(frames[:2], [K, K])
    finally:
        e.cfg['device_glue'] = was
    for k in ('det_position', 'det_scale_r2q', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores', 'det_que_img'):
        np.testing.assert_array_equal(inter[k], want[k], err_msg=k)
    d = float(np.abs(poses - want_poses).max())
    print('first tracked step vs predict_batch, max |dpose|', d)
    assert d <= 1e-6 and len(inter['refine_poses']) == e.cfg['refine_iter'] + 1
    assert inter['bbox_pts'].shape == (2, 8, 2) and inter['smoothed_pts'].shape == (2, 8, 2) and smoothed.shape == (2, 3, 4)


def test_free_running_sequence(est, video):
    """est.track over the 8 frames (predict.py's loop): replay-deterministic, finite, and its smoothed poses are what the
    host twin makes of its own raw poses."""
    from gen6d_b200 import track as T
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    frames, K = video
    was = _set_glue(e, True)
    try:
        a = e.track(frames, K)
        b = e.track(frames, K)
        # one tracked step = one replay of one captured stage and one read of its packed result
        trk = e.tracker()
        trk.step(frames[:1], [K])
        trk.step(frames[1:2], [K])
        k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
        trk.step(frames[2:3], [K])
        stage = [s for key, s in trk.stages.stages.items() if key[0].startswith('track_refine')]
        assert len(stage) == 1 and REPLAYED_KERNELS[0] - k0 == stage[0].kernels
        assert IO_BYTES['d2h'] - d0 == stage[0].static_out[0].numel()
        e.cfg['device_glue'] = False
        h = e.track(frames, K)
    finally:
        e.cfg['device_glue'] = was
    raw = np.stack([r[0] for r in a], 0)
    sm = np.stack([r[1] for r in a], 0)
    np.testing.assert_array_equal(raw, np.stack([r[0] for r in b], 0))
    np.testing.assert_array_equal(sm, np.stack([r[1] for r in b], 0))
    assert np.isfinite(raw).all() and np.isfinite(sm).all()
    ring, count = np.zeros((1, 5, 8, 2), np.float32), np.zeros(1, np.int32)
    worst = 0.0
    for t in range(len(raw)):
        s, _ = T.host_smooth(raw[t][None], True, T.object_bbox(e.refiner.ref_database), K[None], ring, count, T.smoothing_weights(5, 2.5))
        worst = max(worst, float(np.abs(s[0] - sm[t]).max() / np.abs(s[0]).max()))
    assert worst <= 1e-12
    dh = np.abs(raw.astype(np.float64) - np.stack([r[0] for r in h], 0)).reshape(len(raw), -1).max(1)
    print('free-running device graph vs host path, max |dpose| per frame', dh)
    print('free-running vs reference raw poses, max |dR| per frame',
          np.abs(raw[:, :, :3] - TG['track.raw_poses'][:, :, :3]).reshape(len(raw), -1).max(1))


def test_lockstep_sequences_equal_single_sequences(est, video):
    e, _ = est
    frames, K = video
    was = _set_glue(e, True)
    try:
        trk = e.tracker(num_sequences=3)
        trk.start(TG['track.raw_poses'][0:3])
        many, sm_many, _ = trk.step(frames[1:4], [K, K, K])
        one = []
        for s in range(3):
            t1 = e.tracker(num_sequences=1)
            t1.start(TG['track.raw_poses'][s][None])
            one.append(t1.step([frames[s + 1]], [K])[0][0])
    finally:
        e.cfg['device_glue'] = was
    d = float(np.abs(many - np.stack(one, 0)).max())
    print('3 sequences in lockstep vs one at a time, max |dpose|', d)
    assert d <= 2e-4


def test_tracker_errors():
    from gen6d_b200.synthetic import build_estimator, synthetic_database
    e, db = build_estimator()
    K = db.get_K('0')
    for kw in ({'smooth_num': 0}, {'smooth_std': 0.0}, {'smooth_std': -1.0}, {'refine_iter': 0}, {'num_sequences': 0},
               {'bbox_3d': np.zeros((8, 3), np.float32)}):
        with pytest.raises(ValueError):
            e.tracker(**kw)
    trk = e.tracker(num_sequences=2)
    with pytest.raises(ValueError):
        trk.step([db.get_image('0')], [K])
    with pytest.raises(ValueError):
        trk.start(np.zeros((1, 3, 4), np.float32))
    refine_iter = e.cfg['refine_iter']
    trk.step([db.get_image('0'), db.get_image('1')], [K, K])
    trk.step([db.get_image('0'), db.get_image('1')], [K, K])
    assert e.cfg['refine_iter'] == refine_iter                       # tracking never rewrites the estimator's cfg
    e.build(synthetic_database(seed=8), 'all')
    with pytest.raises(RuntimeError, match='stale'):
        trk.step([db.get_image('0'), db.get_image('1')], [K, K])
    trk2 = e.tracker()
    e.selector.load_state_dict(e.selector.state_dict())
    with pytest.raises(RuntimeError, match='stale'):
        trk2.step([db.get_image('0')], [K])
