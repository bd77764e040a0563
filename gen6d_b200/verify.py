"""Checking tracked poses with the detector (row f20).

A refine-only tracking step refines from the previous pose whatever the frame shows.  To tell whether a pose still sits
on the object, the pose is turned back into the detection record that would have produced it (g6d_verify_windows: the
projected object centre c and the scale s = scale_r2q, the inverse of g6d_glue_initial_poses), a window of
WINDOW_FACTOR x ref_resolution pixels is cut there with the selector's detection-crop glue (the object at its reference
size in the middle), the estimator's detector runs on the windows, and g6d_verify_judge maps its detection back to the
frame and judges the row lost: an invalid record, a score below lost_score, or an offset from c above lost_gate
(in reference sizes at the pose's scale).

Gen6DEstimator.verify_poses / ObjectSet.verify_poses run this as one captured graph; the trackers' verify_every replays
a verifying variant of the refine graph (the unchanged refine body, then these nodes, packed into the same read) and
re-initialise the sequences judged lost (Schedule).  The instance trackers' verify_every (row f21) runs the same nodes
over every slot row, M row groups per object."""
import math

import numpy as np
import torch

from . import _lib
from . import glue
from . import ops

WINDOW_FACTOR = 2
_F64_PER_ROW = 5 + 1 + 4             # judge output, lost, window record


def check_thresholds(lost_score, lost_gate):
    """-> (lost_score, lost_gate) as floats or None (the graph key); ValueError for NaN, non-numbers or a negative gate."""
    out = []
    for name, v in (('lost_score', lost_score), ('lost_gate', lost_gate)):
        if v is None:
            out.append(None)
            continue
        try:
            f = float(v)
        except (TypeError, ValueError):
            raise ValueError(f'{name} must be a number or None, got {v!r}') from None
        if math.isnan(f):
            raise ValueError(f'{name} is NaN; pass a number, or None for no threshold')
        out.append(f)
    if out[1] is not None and out[1] < 0:
        raise ValueError(f'lost_gate must be >= 0 (an offset in reference sizes), got {out[1]}')
    return tuple(out)


def graph_name(base, key):
    """The name of the verifying variant of graph `base` with thresholds `key`: apart from every non-verifying name."""
    return ('verify', base) + tuple(key)


def window_size(est):
    return WINDOW_FACTOR * int(est.cfg['ref_resolution'])


def nodes(est, refs, detects, key, M=1):
    """The verification nodes for K objects: fn(frames u8 [qn,h,w,3], cams f64 [qn,20], poses f64 [M*K*qn,12],
    poses_are_f32) -> one float64 tensor [M*K*qn, 10] (judge output, lost, window record).  Row g*qn + s is row group
    g = m*K + o (an instance tracker's slot m of object o; M = 1: object o) on frame s.  refs[o]: object o's
    g6d_glue_refs; detects[o](windows u8 [n,W,W,3]) -> det [n,4]: the detector against object o's references only, run
    once per object over its M*qn windows.  Each window is cut from its own row's frame: the warp jobs of the object's M
    groups point into the same frames, so no frame is copied."""
    W, res = window_size(est), float(est.cfg['ref_resolution'])
    K = len(detects)
    groups = list(refs) * M                        # group m*K + o: object o's refs

    def fn(frames, cams, poses, poses_are_f32):
        qn = frames.shape[0]
        rec = ops.verify_windows(groups, cams, poses, poses_are_f32)
        dets = []
        for o, detect in enumerate(detects):
            jobs = [ops.glue_detection_jobs(rec[g * qn:(g + 1) * qn], frames, W) for g in range(o, M * K, K)]
            jobs = jobs[0] if M == 1 else torch.cat(jobs)
            dets.append(detect(ops.warp_affine_u8(jobs, M * qn, W, W)))
        if K == 1:
            det = dets[0]
        elif M == 1:
            det = torch.cat(dets, 0)
        else:                                      # object-major per group -> row order (m*K + o)*qn + s
            det = torch.stack([d.view(M, qn, 4) for d in dets], 1).reshape(M * K * qn, 4)
        out, lost = ops.verify_judge(rec, det, W, res, *key)
        return torch.cat([out.to(torch.float64), lost.to(torch.float64)[:, None], rec.to(torch.float64)], 1)
    return fn


def packed_bytes(n):
    """Bytes of the verification results of n rows at the end of a step's read."""
    return n * _F64_PER_ROW * 8


def decode(f64, n):
    """The float64 values of nodes()' output, n rows -> verify_poses' result dict."""
    v = np.asarray(f64, np.float64).reshape(n, _F64_PER_ROW)
    out, lost, rec = v[:, :5].astype(np.float32), v[:, 5] != 0, v[:, 6:].astype(np.float32)
    return {'position': out[:, :2].copy(), 'scale': out[:, 2].copy(), 'score': out[:, 3].copy(), 'offset': out[:, 4].copy(),
            'lost': lost, 'window_center': rec[:, :2].copy(), 'window_scale': rec[:, 2].copy()}


def verifying(body, verify):
    """A step body fn(frames, cams, prev, ring, count, *rest) -> (bytes, poses, ring, count) -> the same body followed by
    verify(frames, cams, poses, True) on its final (float32) poses, whose results are appended to the bytes read."""
    def fn(frames, cams, prev, ring, count, *rest):
        buf, poses, ring_o, count_o = body(frames, cams, prev, ring, count, *rest)
        return torch.cat([buf, verify(frames, cams, poses, True).reshape(-1).view(torch.uint8)]), poses, ring_o, count_o
    return fn


def split(host, n):
    """A verifying step's read -> (the step's own bytes, verify_poses' dict of its n rows)."""
    nb = packed_bytes(n)
    return host[:len(host) - nb], decode(host[len(host) - nb:].view(np.float64), n)


# ------------------------------------------------------------------------------------------ the tracker policy
class Schedule:
    """A tracker's verification policy.  Per sequence the tracker keeps `since` (int64 [S]), the refine steps taken since
    its last full prediction, start(), reset() or verification.  A refine step in which a stepped sequence's count reaches
    `every` verifies every stepped sequence and restarts their counts; full and mixed steps never verify, and their
    refining rows still count."""

    def __init__(self, every=None, lost_score=None, lost_gate=None):
        if every is None:
            if lost_score is not None or lost_gate is not None:
                raise ValueError('lost_score / lost_gate judge the verification: pass verify_every too')
        elif not isinstance(every, (int, np.integer)) or isinstance(every, bool) or every < 1:
            raise ValueError(f'verify_every must be an integer >= 1 or None, got {every!r}')
        self.every = None if every is None else int(every)
        self.key = check_thresholds(lost_score, lost_gate)
        self.resets = self.key != (None, None)          # thresholds None: verify and report, never reset

    def due(self, kind, since):
        """Does a step of `kind` over sequences with these counts verify?"""
        return kind == 'refine' and self.due_rows(since, np.ones(len(np.asarray(since)), bool))

    def due_rows(self, since, refining):
        """Does a step of any kind verify whose stepped sequences have counts `since`, of which those in `refining` do not
        re-detect on it?  (The instance trackers, row f21: a step verifies when a refining sequence reaches `every`.)"""
        since = np.asarray(since)[np.asarray(refining, bool)]
        return self.every is not None and bool((since + 1 >= self.every).any())

    @staticmethod
    def advance(since, seqs, pending, verified):
        """Update the counts `since` (in place) after a step over `seqs` whose rows were pending (a full prediction) where
        `pending`."""
        seqs, pending = np.asarray(seqs, np.int64), np.asarray(pending, bool)
        since[seqs[pending]] = 0
        since[seqs[~pending]] += 1
        if verified:
            since[seqs] = 0

    def lost_sequences(self, seqs, lost):
        """The sequences to re-initialise after a verifying step: lost[i] for sequence seqs[i] (any object), none when
        no threshold is set."""
        return np.asarray(seqs, np.int64)[np.asarray(lost, bool)] if self.resets else np.zeros(0, np.int64)


# ------------------------------------------------------------------------------------------ host twins (tests)
def host_windows(poses, poses_are_f32, refs_list, cams):
    """g6d_verify_windows_host: poses [K*qn,3,4] object-major, refs_list[o] a glue.selector_refs dict (numpy), cams
    [qn,20] (glue.cameras) -> records float32 [K*qn,4]."""
    K, cams = len(refs_list), np.ascontiguousarray(cams, np.float64)
    qn = len(cams)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 12))
    if len(p) != K * qn:
        raise ValueError(f'host_windows: {len(p)} poses for {K} objects x {qn} frames')
    keep = [{k: np.ascontiguousarray(r[k], np.float64) for k in ('poses', 'cen', 'f', 'dist', 'center')} for r in refs_list]
    refs = (_lib.GlueRefs * K)(*[glue.refs_struct(r) for r in keep])
    rec = np.zeros((K * qn, 4), np.float32)
    _lib.check(_lib.lib().g6d_verify_windows_host(p.ctypes.data, int(poses_are_f32), refs, K, qn, cams.ctypes.data, rec.ctypes.data),
               'g6d_verify_windows_host')
    return rec


def host_judge(rec, det, window, ref_resolution, lost_score=None, lost_gate=None):
    """g6d_verify_judge_host -> (out float32 [n,5], lost int32 [n])."""
    rec, det = np.ascontiguousarray(rec, np.float32), np.ascontiguousarray(det, np.float32)
    n = len(rec)
    out, lost = np.zeros((n, 5), np.float32), np.zeros(n, np.int32)
    _lib.check(_lib.lib().g6d_verify_judge_host(rec.ctypes.data, det.ctypes.data, n, int(window), float(ref_resolution),
                                                int(lost_score is not None), float(lost_score or 0.0), int(lost_gate is not None),
                                                float(lost_gate or 0.0), out.ctypes.data, lost.ctypes.data),
               'g6d_verify_judge_host')
    return out, lost
