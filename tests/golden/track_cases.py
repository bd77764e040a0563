"""Seeded inputs of the video-tracking goldens (make_golden_track.py) and tests: the camera path of the tracked
sequence and the random pose histories of the smoothing-only set.  Pure functions of their arguments, so the same
poses are rebuilt on any machine; only the reference's outputs are committed (track_golden.npz)."""
import numpy as np


def track_case(query_pose, T=8):
    """Ground-truth poses of a short synthetic video (predict.py's tracking mode): frame 0 is `query_pose` (the estimator
    case's margin-checked query view), every later frame turns the object 1.5 degrees about a fixed axis through its
    centre (the origin) and moves it slightly, a smooth camera path."""
    axis = np.array([0.3, 1.0, 0.2])
    axis /= np.linalg.norm(axis)
    step_t = np.array([0.012, -0.008, 0.03])
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    poses = []
    for t in range(T):
        a = np.deg2rad(1.5) * t
        Rt = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
        R = query_pose[:, :3].astype(np.float64) @ Rt
        poses.append(np.concatenate([R, (query_pose[:, 3].astype(np.float64) + t * step_t)[:, None]], 1))
    return np.stack(poses, 0).astype(np.float32)


def smoothing_case(seed, L=12):
    """A random box, camera and pose history of L frames for the smoothing-only golden set: a slowly moving pose with
    jitter of a few pixels on the projected corners."""
    rng = np.random.RandomState(seed)
    ext, c = rng.uniform(0.4, 2.0, 3), rng.randn(3) * 0.2
    pts = np.stack([c - ext / 2, c + ext / 2]).astype(np.float32)
    f = rng.uniform(400, 1000)
    K = np.array([[f, 0, rng.uniform(280, 360)], [0, f, rng.uniform(200, 280)], [0, 0, 1]], np.float32)
    v = rng.randn(3) * 1.5
    t0 = np.array([rng.randn() * 0.3, rng.randn() * 0.3, rng.uniform(4, 8)])
    dv, dt = rng.randn(3) * 0.01, rng.randn(3) * 0.01
    poses = []
    for k in range(L):
        w = v + k * dv + rng.randn(3) * 0.004           # ~0.25 deg of rotation jitter
        a = np.linalg.norm(w)
        Kx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / a
        R = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
        t = t0 + k * dt + rng.randn(3) * np.array([0.003, 0.003, 0.02])
        poses.append(np.concatenate([R, t[:, None]], 1))
    return {'pts': pts, 'K': K, 'poses': np.stack(poses, 0).astype(np.float32)}
