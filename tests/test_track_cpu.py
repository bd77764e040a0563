"""CPU checks of the tracking smoothing (csrc/track_math.cuh through g6d_track_smooth_host, no GPU): predict.py's box
projection, weighted corner average and PnP against the unmodified reference's functions (track_golden.npz) and
against live cv2.solvePnP(SOLVEPNP_ITERATIVE), and the argument checks of the C ABI."""
import ctypes as C
import os

import numpy as np
import pytest

from gen6d_b200 import _lib
from gen6d_b200 import track as T

HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))


@pytest.fixture(scope='module', autouse=True)
def built():
    from gen6d_b200.build import build
    return build()


def _spacing_ulps(got, want):
    """|got - want| in float32 ulps of the coordinate scale (per column: the largest |u| resp. |v| of the frame)."""
    scale = np.spacing(np.abs(want).max(-2, keepdims=True).astype(np.float32))
    return float((np.abs(got.astype(np.float64) - want) / scale).max())


def _pose_close(got, want, bound=1e-7):
    dR = float(np.abs(got[..., :3] - want[..., :3]).max())
    dt = float((np.abs(got[..., 3] - want[..., 3]).max(-1) / np.linalg.norm(want[..., 3], axis=-1)).max())
    return dR, dt, dR <= bound and dt <= bound


def smoothing_keys():
    return sorted({k.rsplit('.', 1)[0] for k in TG.files if k.startswith('smooth.')})


@pytest.mark.parametrize('key', smoothing_keys())
def test_host_smoothing_matches_reference(key):
    """Step a random pose history through the host twin frame by frame, as predict.py's loop does."""
    num, std = int(key.split('.')[1]), float('.'.join(key.split('.')[2:4]))
    bbox, K, poses = TG[key + '.bbox'], TG[key + '.K'], TG[key + '.poses']
    proj, avg, sm = TG[key + '.proj'], TG[key + '.avg'], TG[key + '.smoothed']
    w = T.smoothing_weights(num, std)
    ring, count = np.zeros((1, num, 8, 2), np.float32), np.zeros(1, np.int32)
    worst_ulp, worst = 0.0, (0.0, 0.0)
    for k in range(len(poses)):
        got_sm, got_avg = T.host_smooth(poses[k][None], True, bbox, K[None], ring, count, w)
        assert count[0] == min(k + 1, num)
        newest = ring[0, count[0] - 1]
        worst_ulp = max(worst_ulp, _spacing_ulps(newest, proj[k]))
        if np.array_equal(ring[0, :count[0]], proj[max(0, k + 1 - num):k + 1]):
            np.testing.assert_array_equal(got_avg[0], avg[k])          # identical corners in -> identical average
        else:
            np.testing.assert_allclose(got_avg[0], avg[k], rtol=1e-6)
        dR, dt, ok = _pose_close(got_sm[0], sm[k])
        worst = (max(worst[0], dR), max(worst[1], dt))
        assert ok, (k, dR, dt)
    print(key, 'projection within', worst_ulp, 'ulp; smoothed pose max |dR|', worst[0], 'relative |dt|', worst[1])
    assert worst_ulp <= 2


def test_host_smoothing_of_the_tracked_sequence():
    """The raw poses of the reference's tracking run, smoothed by the host twin (predict.py --num 5 --std 2.5)."""
    num, std = int(TG['track.num']), float(TG['track.std'])
    raw, K, bbox = TG['track.raw_poses'], TG['track.K'], TG['track.bbox']
    ring, count = np.zeros((1, num, 8, 2), np.float32), np.zeros(1, np.int32)
    for k in range(len(raw)):
        sm, avg = T.host_smooth(raw[k][None], raw.dtype == np.float32, bbox, K[None], ring, count, T.smoothing_weights(num, std))
        assert _spacing_ulps(ring[0, count[0] - 1], TG['track.proj'][k]) <= 2
        np.testing.assert_allclose(avg[0], TG['track.avg'][k], rtol=1e-6)
        assert _pose_close(sm[0], TG['track.smoothed'][k])[2]


def test_host_pnp_matches_opencv():
    """The PnP of the smoothing against live cv2.solvePnP(SOLVEPNP_ITERATIVE) on 2000 random boxes, poses and cameras with
    0-3 px of corner noise.  The noisy corners are fed through the history: with weights (1, 0) the average of a two-frame
    history is exactly its older frame."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.RandomState(5)
    worst = (0.0, 0.0)
    for _ in range(2000):
        ext, c = rng.uniform(0.3, 2.0, 3), rng.randn(3) * 0.3
        box = T.bbox_from_points(np.stack([c - ext / 2, c + ext / 2]).astype(np.float32))
        R, _ = cv2.Rodrigues(rng.randn(3, 1) * 2)
        t = np.array([rng.randn() * 0.5, rng.randn() * 0.5, rng.uniform(3, 8)])
        f = rng.uniform(300, 1200)
        K = np.array([[f, 0, rng.uniform(200, 400)], [0, f * rng.uniform(0.9, 1.1), rng.uniform(150, 300)], [0, 0, 1]], np.float32)
        pose = np.concatenate([R, t[:, None]], 1).astype(np.float32)
        ring, count = np.zeros((1, 1, 8, 2), np.float32), np.zeros(1, np.int32)
        _, clean = T.host_smooth(pose[None], True, box, K[None], ring, count, np.ones(1))
        noisy = (clean[0] + rng.uniform(0, 3) * rng.randn(8, 2)).astype(np.float32)
        ring, count = np.zeros((1, 2, 8, 2), np.float32), np.ones(1, np.int32)
        ring[0, 0] = noisy
        sm, avg = T.host_smooth(pose[None], True, box, K[None], ring, count, np.array([1.0, 0.0]))
        np.testing.assert_array_equal(avg[0], noisy.astype(np.float64))
        _, r, tv = cv2.solvePnP(box.astype(np.float64), avg[0], K.astype(np.float64), np.zeros((8, 1)), flags=cv2.SOLVEPNP_ITERATIVE)
        want = np.concatenate([cv2.Rodrigues(r)[0], tv], 1)
        dR, dt, ok = _pose_close(sm[0], want)
        worst = (max(worst[0], dR), max(worst[1], dt))
        assert ok, (dR, dt)
    print('2000 random PnP problems vs cv2.solvePnP: max |dR|', worst[0], 'relative |dt|', worst[1])


def test_weights_are_predict_py_weights():
    w = T.smoothing_weights(5, 2.5)
    assert w.flags.c_contiguous and w[-1] == 1.0 and np.all(np.diff(w) > 0)


def test_degenerate_box_rejected():
    flat = np.array([[0, 0, 0], [1, 2, 0]], np.float32)
    with pytest.raises(ValueError, match='coplanar'):
        T.bbox_from_points(flat)
    with pytest.raises(ValueError):
        T.check_bbox(np.zeros((4, 3), np.float32))


def test_abi_argument_errors():
    l = _lib.lib()
    S, num = 2, 3
    poses = np.zeros((S, 12)); poses[:, [0, 5, 10]] = 1; poses[:, 11] = 5
    box = T.bbox_from_points(np.array([[-1, -1, -1], [1, 1, 1]], np.float32))
    Ks = np.tile(np.array([500., 0, 320, 0, 500, 240, 0, 0, 1]), (S, 1))
    ring, count = np.zeros((S, num, 8, 2), np.float32), np.zeros(S, np.int32)
    w = T.smoothing_weights(num, 2.5)
    sm, avg = np.zeros((S, 12)), np.zeros((S, 8, 2))
    args = [poses.ctypes.data, 0, box.ctypes.data, Ks.ctypes.data, ring.ctypes.data, count.ctypes.data, num, w.ctypes.data, S,
            sm.ctypes.data, avg.ctypes.data]
    assert l.g6d_track_smooth_host(*args) == 0 and count.tolist() == [1, 1]

    def fails(over, msg):
        a = list(args)
        for i, v in over.items():
            a[i] = v
        assert l.g6d_track_smooth_host(*a) == -1
        assert msg in l.g6d_last_error().decode()

    fails({0: None}, 'null pointer')
    fails({9: None}, 'null pointer')
    fails({6: 0}, 'num >= 1')
    fails({8: 0}, 'S >= 1')
    count[1] = num + 1
    fails({}, 'beyond the ring')
    # the device entry checks its arguments before anything is enqueued (no GPU needed to see the refusal)
    assert l.g6d_track_smooth(None, 0, None, None, None, None, num, None, S, None, None, None) == -1
    assert b'null pointer' in l.g6d_last_error()
    assert l.g6d_track_smooth(*args[:6], 0, *args[7:], None) == -1
    assert b'num >= 1' in l.g6d_last_error()
