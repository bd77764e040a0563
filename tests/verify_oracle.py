"""Numpy restatement of the pose checks of row f20 (csrc/glue_math.cuh window_from_pose / verify_judge), written from
their definitions: the window record of a pose (projected object centre, and the scale_r2q that poses_from_similarity
would have needed for the pose's distance) and the judgement of the detector's record on that window.  Every operation
is a float64 (or float32 where stated) numpy scalar operation in the order the C code evaluates it."""
import numpy as np

D = np.float64


def window_from_pose(pose, f32, center, cam, ref_dist, ref_f):
    """pose [12]; f32: read the pose rounded to float32; center [3]; cam: a glue.cameras row [20] -> float32 [4]."""
    P = [D(np.float32(v)) if f32 else D(v) for v in np.asarray(pose, np.float64).reshape(12)]
    c = [D(v) for v in center]
    K, Kinv, f, f_sq = [D(v) for v in cam[:9]], [D(v) for v in cam[9:18]], D(cam[18]), D(cam[19])
    with np.errstate(all='ignore'):
        depth = (P[8] * c[0] + P[9] * c[1] + P[10] * c[2]) + P[11]
        p = [(P[i * 4] * c[0] + P[i * 4 + 1] * c[1] + P[i * 4 + 2] * c[2]) + P[i * 4 + 3] for i in range(3)]
        q = [K[i * 3] * p[0] + K[i * 3 + 1] * p[1] + K[i * 3 + 2] * p[2] for i in range(3)]
        d = q[2]
        if 0 < abs(d) < 1e-4:
            d = D(1e-4)
        px, py = q[0] / d, q[1] / d
        e = [-((P[i] * P[3] + P[4 + i] * P[7]) + P[8 + i] * P[11]) - c[i] for i in range(3)]
        que_dist = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
        v = [px, py, D(1.0)]
        b = [Kinv[i * 3] * v[0] + Kinv[i * 3 + 1] * v[1] + Kinv[i * 3 + 2] * v[2] for i in range(3)]
        bx, by = b[0] / b[2], b[1] / b[2]
        n2 = np.sqrt((bx * f) * (bx * f) + (by * f) * (by * f))
        que_f_ray = np.sqrt(f_sq + n2 * n2)
        s = D(ref_dist) * que_f_ray / D(ref_f) / que_dist
        cx, cy, fs = np.float32(px), np.float32(py), np.float32(s)
    if depth > 0 and np.isfinite(cx) and np.isfinite(cy) and np.isfinite(fs) and fs > 0:
        return np.asarray([cx, cy, fs, 1], np.float32)
    return np.asarray([0, 0, 1, 0], np.float32)


def windows(poses, f32, refs_list, cams):
    """Object-major poses [K*qn, 3, 4], refs_list[o] a glue.selector_refs dict, cams [qn,20] -> records float32 [K*qn,4]."""
    qn = len(cams)
    P = np.asarray(poses, np.float64).reshape(-1, 12)
    out = np.zeros((len(P), 4), np.float32)
    for i in range(len(P)):
        r = refs_list[i // qn]
        out[i] = window_from_pose(P[i], f32, r['center'], cams[i % qn], r['dist'][0], r['f'][0])
    return out


def judge(rec, det, window, ref_resolution, lost_score=None, lost_gate=None):
    """rec [n,4], det [n,4] -> (out float32 [n,5], lost int32 [n])."""
    rec, det = np.asarray(rec, np.float32), np.asarray(det, np.float32)
    n = len(rec)
    out, lost = np.zeros((n, 5), np.float32), np.zeros(n, np.int32)
    half = D(window // 2)
    with np.errstate(all='ignore'):
        for i in range(n):
            cx, cy, s = D(rec[i, 0]), D(rec[i, 1]), D(rec[i, 2])
            dx, dy = (D(det[i, 0]) - half) * s, (D(det[i, 1]) - half) * s
            out[i] = [np.float32(cx + dx), np.float32(cy + dy), np.float32(D(det[i, 2]) * s), det[i, 3],
                      np.float32(np.sqrt(dx * dx + dy * dy) / (D(ref_resolution) * s))]
            bad = rec[i, 3] == 0
            if lost_score is not None and not D(out[i, 3]) >= D(lost_score):
                bad = True
            if lost_gate is not None and not D(out[i, 4]) <= D(lost_gate):
                bad = True
            lost[i] = int(bad)
    return out, lost
