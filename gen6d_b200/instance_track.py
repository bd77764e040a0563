"""Multi-instance tracking (Gen6DEstimator.instance_tracker()): every instance of an object followed through S videos in
lockstep, with identities kept across periodic re-detection.

Each sequence has M slots (instances.py's instance-major layout: row m*S + s is slot m of sequence s).  A slot holds a live
track (an id, its previous pose, a miss count, its smoothing ring) or nothing.  Two kinds of step, each ONE captured graph
and one read (instances.pack):

- a re-detection step (the first, the one after reset() / redetect(), and every `redetect_every`-th after the last one)
  runs predict_instances' detection half (the detector's maps, g6d_det_parse_peaks, the M*S crops and selections, the
  initial poses), then g6d_instances_associate: the live tracks are matched greedily to the detections by the distance of
  their projected object centre to the detected position, in units of the detection box; unmatched tracks take a miss
  and are dropped past max_misses, unmatched detections start tracks in the lowest empty slots, and every slot still
  empty parks on detection row m of its frame.  Continuing tracks run `refine_iter` refinements, new tracks and parked
  slots cfg['refine_iter'], through the row-indexed glue (csrc/glue.cu) with scratch rows for finished chains, so every
  iteration is one refiner stage over exactly M*S poses;
- every other step refines every slot `refine_iter` times from its previous pose (an empty slot from its parking pose),
  as Tracker's refine step does for one instance.

Both finish with predict.py's smoothing, slots standing in for the objects of g6d_track_smooth_objects.  Shapes are
fixed, so empty slots are computed too; their results come back as NaN.  The slot state stays on the device.

ObjectInstanceTracker (ObjectSet.instance_tracker()) does the same for every object of an object set at once: slot group
g = m*K + o is instance slot m of object o (row g*S + s, the layout of ObjectSet.predict_instances' slots), the
re-detection step runs the set's shared pyramid and correlation and g6d_instances_associate_objects (each object's
tracks matched against its own peaks, one id counter), and every refinement iteration is still ONE refiner stage over
all M*K*S poses.  Both trackers are the class below, parameterised by the per-group tables and the detection.

Re-detection schedules (row f18, schedule=): 'lockstep' re-detects every sequence on the same steps.  'per_sequence'
gives every sequence its own pending flag and re-detection counter (host-side, so planning a step reads nothing from the
device): reset(sequences) / redetect(sequences) mark only those sequences, and step(..., sequences=[...]) steps any
subset as Tracker.step does (row f17).  'staggered' is 'per_sequence' whose periodic re-detections are spread over the
steps: a detection leaves a sequence's counter at 1 (the lockstep count), except one it was marked for (its first, or
after reset / redetect), which leaves it at 1 + floor(s*E/S); sequence s then re-detects every E steps from E - floor(s*E/S)
steps on, so in lockstep stepping at most ceil(S/E) sequences re-detect on any later step (Schedule).  Each step is still one
graph and one read: with b the stepped batch (all S, or the listed sequences padded to f17's bucket) and d the bucket of
its re-detecting sequences, d = 0 replays the refine body, d = b the re-detection body, and anything between the mixed
instance step (_mixed_fn): the re-detecting sequences' frames are gathered and detected as a batch of d,
g6d_instances_associate_sequences associates them and sets up every other pair's refinement, and the iterations past
refine_iter run one refiner stage over the re-detecting sequences' slots only.

Boxes from another detector (row f19): step(..., boxes=) re-detects from caller boxes instead of the detector.  Their
records (g6d_det_from_boxes) take the place of the peaks in the same bodies, under graph names of their own
(boxes.graph_name) with the box buffer as the last graph input.  Lockstep: boxes for every sequence, and the step is a
re-detection step.  Per-sequence schedules: exactly the stepped sequences given boxes re-detect (the mixed step when only
some do), and their detection counts in the schedule as a detector detection does; a due sequence without boxes is not
detected and stays due.

Verification (row f21, verify_every=): a step verifies when a stepped sequence that does not re-detect on it has taken
verify_every steps since its last re-detection, reset, redetect or verification (verify.Schedule.due_rows); refine and
mixed steps alike.  Its graph is the unchanged step body followed by verify.nodes on the final float32 poses of every slot
row (M*K*S windows, one detector call per object over its M*S windows) and, with a threshold set,
g6d_instances_verify_update: a live slot of a verified sequence judged lost takes a miss and is dropped past max_misses
as the association drops an unmatched track, one judged found restarts its misses.  Everything lands in the same read,
under verify.graph_name.  The sequences with a lost slot then re-detect on their next step ('lockstep': every sequence),
so the association can correct a wrong verdict and a track it matches keeps its id.
"""
import numpy as np
import torch

from . import _lib
from . import boxes as B
from . import draw as dr
from . import frames as fr
from . import glue
from . import instances
from . import ops
from . import verify as V
from .graphs import StageCache
from .track import (PartialStep, _bucket, _gather_rows, _scatter_rows, _sequences, _size_buckets, check_bbox, draw_inputs,
                    object_bbox, object_bboxes, smoothing_weights)


def staggered_phases(S, E):
    """Each sequence's phase under schedule='staggered': floor(s*E/S) for sequence s."""
    return (np.arange(S) * int(E)) // int(S)


class Schedule:
    """The host plan of a per-sequence schedule (row f18): per sequence a pending flag (marked by the first step, reset and
    redetect) and `count`, the steps since its last detection counting the step of that detection as 1, as the lockstep
    tracker counts.  A sequence re-detects when pending or when count >= E (redetect_every).  After a detection it was
    marked for, its count restarts at 1 + phase (phase 0 under 'per_sequence', floor(s*E/S) under 'staggered', so a
    sequence of phase p re-detects periodically E - p steps later); after a periodic one, at 1."""

    def __init__(self, S, E, staggered):
        self.S, self.E = S, E
        self.pending, self.count = np.ones(S, bool), np.zeros(S, np.int64)
        self.phase = staggered_phases(S, E) if staggered else np.zeros(S, np.int64)

    def due(self):
        """bool [S]: the sequences that re-detect on their next step."""
        return self.pending | ((self.count >= self.E) if self.E is not None else False)

    def plan(self, seqs, n_real, hit=None):
        """The stepped batch seqs [b] (its first n_real rows real, the rest padding) -> (det_seq bool [b], kind): the rows
        that re-detect (padding never does, so it spawns no ids) and the body the step runs ('refine': none, 'detect':
        every row, else 'mixed').  hit bool [b]: the rows that re-detect whether due or not (a step with boxes: the rows
        given boxes); None: the due rows."""
        det_seq = self.due()[seqs] if hit is None else np.array(hit, bool)
        det_seq[n_real:] = False
        m = int(det_seq.sum())
        return det_seq, 'refine' if m == 0 else 'detect' if m == len(seqs) else 'mixed'

    def advance(self, stepped, hit=None):
        """The counters after a step of the distinct sequences `stepped`, of which those in hit (bool, aligned; None: the
        due ones) re-detected.  A sequence that re-detected counts as a detection; any other, due or not, as a step
        without one (a due sequence stays due)."""
        hit = self.due()[stepped] if hit is None else np.asarray(hit, bool)
        restart = self.pending[stepped] & hit
        self.count[stepped] = np.where(hit, np.where(restart, 1 + self.phase[stepped], 1), self.count[stepped] + 1)
        self.pending[stepped[hit]] = False


def plan_mixed(det_seq, plan):
    """A mixed step's detection batch -> (gathered sequences [d], per-size blocks or None, det_index [b] (each sequence's
    row in the batch, -1: none), d, the graph key of the batch).  One size: the re-detecting sequences ascending, padded to
    d = _bucket(m, b) by repeating the last; several sizes (plan.mixed): _size_buckets' per-size blocks."""
    S, det = len(det_seq), np.flatnonzero(det_seq)
    if plan is not None and plan.mixed:
        seq, blocks, pick = _size_buckets(det, plan)
        d, key = len(seq), tuple(blocks)
    else:
        d = _bucket(len(det), S)
        seq, blocks, pick, key = np.concatenate([det, np.full(d - len(det), det[-1])]), None, np.arange(len(det)), d
    det_index = np.full(S, -1, np.int64)
    det_index[det] = pick
    check_det_index(det_index, S, d)
    return seq, blocks, det_index, d, key


def mixed_name(b, key):
    """The graph name of the mixed instance step over b sequences with detection batch `key` (d, or per-size blocks)."""
    return ('instance_mixed', b, key)


def host_associate(det, valid, init, cams, center, ref_resolution, gate, max_misses, F, r, prev, live, ids, misses, next_id,
                   park, ring, count):
    """g6d_instances_associate_host on numpy arrays (the shapes and dtypes of ops.instances_associate; cams float64 [S,20]).
    live, ids, misses, next_id, park, ring and count are updated in place.  Returns (work, flags0, lists, det_slot, spawned,
    dropped) as numpy arrays."""
    n, S = len(live), len(cams)
    M, num = n // S, ring.shape[1]
    for a, dt in ((live, np.int32), (ids, np.int64), (misses, np.int32), (next_id, np.int64), (park, np.float64),
                  (ring, np.float32), (count, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_associate: the state arrays must be contiguous {dt.__name__} arrays (updated in place)')
    c = lambda a, dt: np.ascontiguousarray(a, dt)
    det, valid, init, cams, prev = c(det, np.float32), c(valid, np.int32), c(init, np.float64), c(cams, np.float64), c(prev, np.float64)
    work, flags0 = np.zeros((2 * n, 12)), np.zeros(2 * n, np.uint8)
    lists = np.zeros(max(F, r) * n, np.int32)
    det_slot, spawned, dropped = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int64)
    cx, cy, cz = (float(v) for v in center)
    _lib.check(_lib.lib().g6d_instances_associate_host(
        S, M, int(F), int(r), det.ctypes.data, valid.ctypes.data, init.ctypes.data, cams.ctypes.data, cx, cy, cz,
        float(ref_resolution), float(gate), int(max_misses), prev.ctypes.data, live.ctypes.data, ids.ctypes.data,
        misses.ctypes.data, next_id.ctypes.data, park.ctypes.data, ring.ctypes.data, count.ctypes.data, num,
        work.ctypes.data, flags0.ctypes.data, lists.ctypes.data, det_slot.ctypes.data, spawned.ctypes.data,
        dropped.ctypes.data), 'g6d_instances_associate_host')
    return work, flags0, lists, det_slot, spawned, dropped


def host_associate_objects(det, valid, init, cams, centers, ref_resolution, gate, max_misses, F, r, prev, live, ids, misses,
                           next_id, park, ring, count):
    """g6d_instances_associate_objects_host on numpy arrays (the shapes and dtypes of ops.instances_associate_objects;
    centers float64 [K,3], cams float64 [S,20]).  live, ids, misses, next_id, park, ring and count are updated in place.
    Returns (work, flags0, lists, det_slot, spawned, dropped) as numpy arrays."""
    c = lambda a, dt: np.ascontiguousarray(a, dt)
    centers = c(centers, np.float64).reshape(-1, 3)
    n, S, K = len(live), len(cams), len(centers)
    M, num = n // max(K * S, 1), ring.shape[1]
    for a, dt in ((live, np.int32), (ids, np.int64), (misses, np.int32), (next_id, np.int64), (park, np.float64),
                  (ring, np.float32), (count, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_associate_objects: the state arrays must be contiguous {dt.__name__} arrays (updated in place)')
    det, valid, init, cams, prev = c(det, np.float32), c(valid, np.int32), c(init, np.float64), c(cams, np.float64), c(prev, np.float64)
    work, flags0 = np.zeros((2 * n, 12)), np.zeros(2 * n, np.uint8)
    lists = np.zeros(max(F, r) * n, np.int32)
    det_slot, spawned, dropped = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int64)
    _lib.check(_lib.lib().g6d_instances_associate_objects_host(
        S, K, M, int(F), int(r), det.ctypes.data, valid.ctypes.data, init.ctypes.data, cams.ctypes.data, centers.ctypes.data,
        float(ref_resolution), float(gate), int(max_misses), prev.ctypes.data, live.ctypes.data, ids.ctypes.data,
        misses.ctypes.data, next_id.ctypes.data, park.ctypes.data, ring.ctypes.data, count.ctypes.data, num,
        work.ctypes.data, flags0.ctypes.data, lists.ctypes.data, det_slot.ctypes.data, spawned.ctypes.data,
        dropped.ctypes.data), 'g6d_instances_associate_objects_host')
    return work, flags0, lists, det_slot, spawned, dropped


def host_verify_update(lost, verified, max_misses, live, ids, misses):
    """g6d_instances_verify_update_host on numpy arrays: lost, verified int [n]; live int32, ids int64 and misses int32
    [n] are updated in place.  Returns dropped int64 [n]."""
    for a, dt in ((live, np.int32), (ids, np.int64), (misses, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_verify_update: the state arrays must be contiguous {dt.__name__} arrays (updated in place)')
    lost, verified = np.ascontiguousarray(lost, np.int32), np.ascontiguousarray(verified, np.int32)
    dropped = np.zeros(len(live), np.int64)
    _lib.check(_lib.lib().g6d_instances_verify_update_host(len(live), lost.ctypes.data, verified.ctypes.data, int(max_misses),
                                                           live.ctypes.data, ids.ctypes.data, misses.ctypes.data,
                                                           dropped.ctypes.data), 'g6d_instances_verify_update_host')
    return dropped


def check_det_index(det_index, S, D):
    """ValueError unless det_index [S] holds -1 (the sequence does not detect) or distinct rows j < D, with 0 <= D <= S."""
    det_index = np.asarray(det_index).reshape(-1)
    if len(det_index) != S or not 0 <= int(D) <= S:
        raise ValueError(f'det_index: need {S} entries and 0 <= D <= {S}, got {len(det_index)} entries and D = {D}')
    bad = det_index[(det_index < -1) | (det_index >= D)]
    if len(bad):
        raise ValueError(f'det_index: entries {bad.tolist()} are outside [-1, {D})')
    rows = det_index[det_index >= 0]
    if len(np.unique(rows)) != len(rows):
        raise ValueError(f'det_index: {det_index.tolist()} lists a detection row twice')


def list_length(G, S, D, F, r):
    """Entries of the row lists of g6d_instances_associate_sequences for G slot groups: r iterations over every row, then
    max(F - r, 0) over the detecting sequences' D rows per group."""
    return r * G * S + max(F - r, 0) * G * D


def host_associate_sequences(det_index, det, valid, init, cams, centers, ref_resolution, gate, max_misses, F, r, prev, live, ids,
                             misses, next_id, park, ring, count):
    """g6d_instances_associate_sequences_host on numpy arrays: det_index int [S] (-1: the sequence does not detect, else its
    row j < D in the detection batch; D = len(det) // (M*K)), det [M*K*D,4], valid [M*K*D], init [M*K*D,12], the rest as
    host_associate_objects.  live, ids, misses, next_id, park, ring and count are updated in place.  Returns (work, flags0,
    lists, det_slot, spawned, dropped) as numpy arrays."""
    c = lambda a, dt: np.ascontiguousarray(a, dt)
    centers = c(centers, np.float64).reshape(-1, 3)
    n, S, K = len(live), len(cams), len(centers)
    G, num = n // max(K * S, 1) * K, ring.shape[1]
    D = len(det) // max(G, 1)
    for a, dt in ((live, np.int32), (ids, np.int64), (misses, np.int32), (next_id, np.int64), (park, np.float64),
                  (ring, np.float32), (count, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_associate_sequences: the state arrays must be contiguous {dt.__name__} arrays (updated in place)')
    det_index, det, valid, init = c(det_index, np.int32), c(det, np.float32), c(valid, np.int32), c(init, np.float64)
    cams, prev = c(cams, np.float64), c(prev, np.float64)
    work, flags0 = np.zeros((2 * n, 12)), np.zeros(2 * n, np.uint8)
    lists = np.zeros(list_length(G, S, D, int(F), int(r)), np.int32)
    det_slot, spawned, dropped = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int64)
    _lib.check(_lib.lib().g6d_instances_associate_sequences_host(
        S, K, n // max(K * S, 1), int(F), int(r), D, det_index.ctypes.data, det.ctypes.data, valid.ctypes.data, init.ctypes.data,
        cams.ctypes.data, centers.ctypes.data, float(ref_resolution), float(gate), int(max_misses), prev.ctypes.data,
        live.ctypes.data, ids.ctypes.data, misses.ctypes.data, next_id.ctypes.data, park.ctypes.data, ring.ctypes.data,
        count.ctypes.data, num, work.ctypes.data, flags0.ctypes.data, lists.ctypes.data, det_slot.ctypes.data,
        spawned.ctypes.data, dropped.ctypes.data), 'g6d_instances_associate_sequences_host')
    return work, flags0, lists, det_slot, spawned, dropped


SCHEDULES = ('lockstep', 'per_sequence', 'staggered')


def check_args(num_sequences, max_instances, refine_iter, redetect_every, gate, max_misses, min_score, nms_iou, peak_radius,
               smooth_num, smooth_std, schedule='lockstep'):
    """-> the detection key of instances.check_args; ValueError for a bad argument."""
    key = instances.check_args(max_instances, nms_iou, peak_radius, min_score)
    if schedule not in SCHEDULES:
        raise ValueError(f'schedule={schedule!r}: need one of {SCHEDULES}')
    if schedule == 'staggered' and redetect_every is None:
        raise ValueError("schedule='staggered' spreads the periodic re-detections: it needs redetect_every")
    if int(num_sequences) < 1:
        raise ValueError(f'num_sequences must be >= 1, got {num_sequences}')
    if int(refine_iter) < 1:
        raise ValueError(f'refine_iter must be >= 1, got {refine_iter}')
    if redetect_every is not None and int(redetect_every) < 1:
        raise ValueError(f'redetect_every must be None or >= 1, got {redetect_every}')
    if not (np.isfinite(float(gate)) and float(gate) > 0):
        raise ValueError(f'gate must be finite and > 0, got {gate}')
    if int(max_misses) < 0:
        raise ValueError(f'max_misses must be >= 0, got {max_misses}')
    if int(smooth_num) < 1:
        raise ValueError(f'smooth_num must be >= 1, got {smooth_num}')
    if not float(smooth_std) > 0:
        raise ValueError(f'smooth_std must be > 0, got {smooth_std}')
    return key


class InstanceTracker:
    """Every instance of the estimator's object tracked through S sequences in lockstep; see Gen6DEstimator.instance_tracker().

    The state, the two graph bodies, reset and the decode are written for K objects with M slots each (K = 1 here); a
    subclass supplies the per-group tables (_groups), the detection (_detection), the id association (_associate) and the
    readback of the selections (_take_selections)."""

    _verify = V.Schedule()           # no verification (row f21)

    def __init__(self, est, num_sequences, max_instances=4, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1,
                 min_score=None, nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5, bbox_3d=None, draw=None,
                 draw_color=dr.DEFAULT_COLOR, schedule='lockstep', verify_every=None, lost_score=None, lost_gate=None):
        from .objects import require_device_pipeline
        require_device_pipeline(est, 'instance tracking')
        key = check_args(num_sequences, max_instances, refine_iter, redetect_every, gate, max_misses, min_score, nms_iou,
                         peak_radius, smooth_num, smooth_std, schedule)
        verify = V.Schedule(verify_every, lost_score, lost_gate)
        if bbox_3d is None:
            bbox_3d = object_bbox(est.refiner.ref_database)
            if bbox_3d is None:
                raise ValueError('the database has no object point cloud: pass bbox_3d (the 8 corners of the object box)')
        self.bbox = check_bbox(bbox_3d)
        self._gen = est._generation()
        self._setup(est, key, [self.bbox], num_sequences, refine_iter, redetect_every, gate, max_misses, smooth_num, smooth_std,
                    draw, [draw_color], schedule, verify)
        center = np.asarray(est.ref_info['center'], np.float64).reshape(1, 3)
        self._dev['centers'] = torch.from_numpy(np.ascontiguousarray(center)).to(est.detector.device)

    def _setup(self, est, key, boxes, num_sequences, refine_iter, redetect_every, gate, max_misses, smooth_num, smooth_std,
               draw=None, colors=None, schedule='lockstep', verify=None):
        """The tracker's constants and device state for K = len(boxes) objects with M = key[0] slots each; verify: a
        verify.Schedule (row f21)."""
        self.est, self.key, self.schedule = est, key, schedule
        self.K, self.S, self.M, self.refine_iter = len(boxes), int(num_sequences), key[0], int(refine_iter)
        self.redetect_every = None if redetect_every is None else int(redetect_every)
        self.gate, self.max_misses = float(gate), int(max_misses)
        self.num, self.std = int(smooth_num), float(smooth_std)
        self.weights = smoothing_weights(self.num, self.std)
        self.stages = StageCache()       # the detect and refine graphs (they capture this tracker's device state)
        dev = est.detector.device
        groups = np.ascontiguousarray(np.tile(np.stack(boxes, 0), (self.M, 1, 1)))       # group m*K + o smooths with box o
        self._dev = {'bboxes': torch.from_numpy(groups).to(dev), 'weights': torch.from_numpy(self.weights.copy()).to(dev)}
        n = self.M * self.K * self.S
        self._next_id = torch.zeros(1, dtype=torch.int64, device=dev)     # ids are unique over the tracker's life
        self._state = {'prev': torch.zeros(n, 12, dtype=torch.float64, device=dev),
                       'park': torch.zeros(n, 12, dtype=torch.float64, device=dev),
                       'live': torch.zeros(n, dtype=torch.int32, device=dev),
                       'ids': torch.full((n,), -1, dtype=torch.int64, device=dev),
                       'misses': torch.zeros(n, dtype=torch.int32, device=dev),
                       'ring': torch.zeros(n, self.num, 8, 2, dtype=torch.float32, device=dev),
                       'count': torch.zeros(n, dtype=torch.int32, device=dev)}
        self._pending, self._since = True, 0
        # per-sequence schedules (row f18): each sequence's pending flag and steps since its last detection, on the host
        self._schedule = Schedule(self.S, self.redetect_every, schedule == 'staggered')
        if verify is not None:
            self._verify = verify
        self._vsince = np.zeros(self.S, np.int64)     # steps since the last re-detection / reset / redetect / verification
        # drawing (row f16): every live slot (track id >= 0) of a sequence on its frame, in row (slot group) order
        kinds = self.draw = dr.parse_kinds(draw)
        G = self.M * self.K
        self._drawer = dr.StepDrawer(kinds, colors, np.stack(boxes, 0), [g % self.K for g in range(G)], self.S, dev,
                                     live=True) if kinds else None

    # -------------------------------------------------------------- state
    def reset(self, sequences=None):
        """Drop the tracks of `sequences` (None: every sequence); the next step re-detects.  Ids are never reused."""
        st = self._state
        if sequences is None:
            rows = slice(None)
        else:
            seqs = _sequences(self.S, sequences)
            rows = torch.from_numpy(np.concatenate([g * self.S + seqs for g in range(self.M * self.K)])).to(st['live'].device)
        st['live'][rows] = 0
        st['ids'][rows] = -1
        st['misses'][rows] = 0
        st['ring'][rows] = 0
        st['count'][rows] = 0
        self._pending = True
        self._schedule.pending[slice(None) if sequences is None else seqs] = True
        if self._verify.every is not None:
            self._vsince[slice(None) if sequences is None else seqs] = 0

    def redetect(self, sequences=None):
        """The next step re-detects: the live tracks are kept and associated with the new detections.  sequences (the
        per-sequence schedules only): mark only those sequences; each re-detects on its next step."""
        if sequences is None:
            self._pending = True
            self._schedule.pending[:] = True
            if self._verify.every is not None:
                self._vsince[:] = 0
            return
        if self.schedule == 'lockstep':
            raise ValueError("redetect(sequences): a lockstep tracker re-detects every sequence together; create it with "
                             "schedule='per_sequence' or 'staggered' to re-detect single sequences")
        seqs = _sequences(self.S, sequences)
        self._schedule.pending[seqs] = True
        if self._verify.every is not None:
            self._vsince[seqs] = 0

    def detecting(self):
        """bool [S]: the sequences that re-detect on their next step."""
        if self.schedule == 'lockstep':
            return np.full(self.S, self._detecting())
        return self._schedule.due()

    def _check(self):
        if self.est._generation() != self._gen:
            raise RuntimeError('this instance tracker is stale: the estimator was rebuilt (build() on another object) or its '
                               'weights changed since the tracker was created; create a new one with est.instance_tracker()')

    def _detecting(self):
        return self._pending or (self.redetect_every is not None and self._since >= self.redetect_every)

    # -------------------------------------------------------------- what differs between the estimator and an object set
    def _tables(self):
        return self.est._glue_state()

    def _groups(self, st):
        """-> (the refiner's view table of every slot group, the reference views per table)."""
        return [st['views']] * self.M, st['tables']['ref_num']

    def _detection(self, st, boxes=None):
        """-> fn(frames, cams) -> (initial poses [n,12], det [n,4], crops, the selections' tensors in packing order, valid
        int32 [n], instance count int32 [K*S]): predict_instances' detection half on the S frames (boxes: a boxes.Detect,
        the detection from caller boxes)."""
        detect, extra = (boxes, boxes.extra) if boxes is not None else self.est._peaks_detect_fn(*self.key)
        initial = self.est._initial_poses_device_fn(st, detect)

        def fn(frames, cams):
            init, det, crop, idx, sel_out, logits = initial(frames, cams)
            return (init, det, crop, [idx, sel_out, logits], *extra)
        return fn

    def _associate(self):
        center = [float(v) for v in np.asarray(self.est.ref_info['center']).reshape(3)]
        return lambda det, valid, init, cams, *state: ops.instances_associate(
            det, valid, init, cams, center, float(self.est.cfg['ref_resolution']), self.gate, self.max_misses,
            self.est.cfg['refine_iter'], self.refine_iter, *state)

    def _take_selections(self, rd, S):
        """-> per object (sel_idx [M*S], sel_out [M*S*2], logits [M*S*n_sel]) instance-major, read in packing order (S:
        the detected frames)."""
        n = self.M * S
        return [(rd.take(n), rd.take(n * 2), rd.take(n * len(self.est.ref_info['poses'])))]

    def _verify_fn(self, st):
        """verify.nodes over the M*K slot groups: each group's windows detected against its object's references."""
        return self.est._verify_fn(st, self._verify.key, self.M)

    # -------------------------------------------------------------- the graphs
    def _detect_fn(self, st, draw=None, S=None, boxes=None):
        """The re-detection body for S sequences (default: the tracker's; a partial step's compact batch, row f18); boxes:
        a boxes.Detect, the detection from caller boxes (row f19)."""
        est, G, S, r = self.est, self.M * self.K, S or self.S, self.refine_iter
        F, c, n = est.cfg['refine_iter'], self._dev, self.M * self.K * S
        views, R = self._groups(st)
        initial, associate, refine = self._detection(st, boxes), self._associate(), est.refiner._refine_warped(128)

        def fn(frames, cams, prev, park, live, ids, misses, next_id, ring, count, *dt):
            init, det, crop, sels, valid, inst_count = initial(frames, cams)
            work, flags0, lists, det_slot, spawned, dropped = associate(det, valid, init, cams, prev, live, ids, misses, next_id,
                                                                        park, ring, count)
            frames_x, cams_x = torch.cat([frames, frames], 0), torch.cat([cams, cams], 0)
            real = lambda: work.view(G, 2 * S, 12)[:, :S].reshape(n, 12).clone()
            ones, chain = torch.ones_like(flags0), [real()]
            for it in range(max(F, r)):
                rows = lists[it * n:(it + 1) * n]
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_rows(
                    views, R, 2 * S, cams_x, frames_x, work, rows, flags0 if it == 0 else ones)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)            # one refiner stage over all n poses
                ops.glue_apply_refinements_rows(views, 2 * S, que_pose, que_K, rect, out, rows, work)
                chain.append(real())
            poses = chain[-1]
            Ks = cams[:, :9].contiguous()
            smoothed, avg = ops.track_smooth_objects(poses, True, c['bboxes'], Ks, ring, count, c['weights'])
            if dt:
                draw(frames, poses, True, smoothed, Ks, dt[0], ids)
            buf = instances.pack([torch.stack(chain, 0), smoothed, avg, ring, count, ids, det, *sels, valid, inst_count, det_slot,
                                  spawned, dropped], crop)
            return buf, poses, park, live, ids, misses, next_id, ring, count
        return fn

    def _refine_fn(self, st, draw=None, S=None):
        est, S, r, c = self.est, S or self.S, self.refine_iter, self._dev
        n = self.M * self.K * S
        views, R = self._groups(st)
        refine = est.refiner._refine_warped(128)

        def fn(frames, cams, prev, park, live, ids, ring, count, *dt):
            work = torch.where((live != 0)[:, None], prev, park)                 # empty slots restart from their parking pose
            flags0 = live.to(torch.uint8)                                        # tracks hold float32 values, parking poses not
            rows = torch.arange(n, device=live.device, dtype=torch.int32)
            ones, chain = torch.ones_like(flags0), [work.clone()]
            for it in range(r):
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_rows(
                    views, R, S, cams, frames, work, rows, flags0 if it == 0 else ones)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)
                ops.glue_apply_refinements_rows(views, S, que_pose, que_K, rect, out, rows, work)
                chain.append(work.clone())
            poses = chain[-1]
            Ks = cams[:, :9].contiguous()
            smoothed, avg = ops.track_smooth_objects(poses, True, c['bboxes'], Ks, ring, count, c['weights'])
            if dt:
                draw(frames, poses, True, smoothed, Ks, dt[0], ids)
            buf = instances.pack([torch.stack(chain, 0), smoothed, avg, ring, count, ids], torch.empty(0, dtype=torch.uint8,
                                                                                                     device=live.device))
            return buf, poses, ring, count
        return fn

    def _mixed_fn(self, st, S, d, blocks=None, draw=None, boxes=None):
        """The mixed instance step's body for S sequences of which some re-detect, their frames gathered into a batch of
        d (blocks: per size group of frames of several sizes, as _size_buckets makes them; boxes: a boxes.Detect over the
        S sequences' maps, gathered like the frames)."""
        est, G, r = self.est, self.M * self.K, self.refine_iter
        F, c, n = est.cfg['refine_iter'], self._dev, self.M * self.K * S
        views, R = self._groups(st)
        initial, refine = self._detection(st, boxes), est.refiner._refine_warped(128)
        ref_res = float(est.cfg['ref_resolution'])

        def fn(frames, cams, prev, park, live, ids, misses, next_id, ring, count, seq, det_index, *dt):
            gf, gc = frames.index_select(0, seq), cams.index_select(0, seq)
            if boxes is not None:
                boxes.select(seq)
            if blocks is None:
                init, det, crop, sels, valid, inst_count = initial(gf, gc)
            else:
                with fr.gathered(frames, gf, seq, blocks):                       # detection on true-size frames (row f13)
                    init, det, crop, sels, valid, inst_count = initial(gf, gc)
            work, flags0, lists, det_slot, spawned, dropped = ops.instances_associate_sequences(
                det_index, det, valid, init, cams, c['centers'], ref_res, self.gate, self.max_misses, F, r, prev, live, ids, misses,
                next_id, park, ring, count)
            frames_x, cams_x = torch.cat([frames, frames], 0), torch.cat([cams, cams], 0)
            real = lambda: work.view(G, 2 * S, 12)[:, :S].reshape(n, 12).clone()
            ones, chain, off = torch.ones_like(flags0), [real()], 0
            for it in range(max(F, r)):
                L = n if it < r else G * d                  # past refine_iter: the re-detecting sequences' slots only
                rows = lists[off:off + L]
                off += L
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_rows(
                    views, R, 2 * S, cams_x, frames_x, work, rows, flags0 if it == 0 else ones)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)
                ops.glue_apply_refinements_rows(views, 2 * S, que_pose, que_K, rect, out, rows, work)
                chain.append(real())
            poses = chain[-1]
            Ks = cams[:, :9].contiguous()
            smoothed, avg = ops.track_smooth_objects(poses, True, c['bboxes'], Ks, ring, count, c['weights'])
            if dt:
                draw(frames, poses, True, smoothed, Ks, dt[0], ids)
            buf = instances.pack([torch.stack(chain, 0), smoothed, avg, ring, count, ids, det, *sels, valid, inst_count, det_slot,
                                  spawned, dropped], crop)
            return buf, poses, park, live, ids, misses, next_id, ring, count
        return fn

    def _body(self, st, kind, S, d=None, blocks=None, draw=None, boxes=None):
        """A per-sequence step's body on the whole slot state: fn(frames, cams, prev, park, live, ids, misses, next_id, ring,
        count, *rest) -> (buf, prev, park, live, ids, misses, next_id, ring, count), kind 'detect', 'refine' or 'mixed'."""
        if kind == 'detect':
            return self._detect_fn(st, draw, S, boxes)
        if kind == 'mixed':
            return self._mixed_fn(st, S, d, blocks, draw, boxes)
        refine = self._refine_fn(st, draw, S)

        def fn(frames, cams, prev, park, live, ids, misses, next_id, ring, count, *dt):
            buf, poses, ring, count = refine(frames, cams, prev, park, live, ids, ring, count, *dt)
            return buf, poses, park, live, ids, misses, next_id, ring, count
        return fn

    def _verifying(self, body, st):
        """A per-sequence step body (_body's signature) -> its verifying variant (row f21): the body unchanged, then
        verify.nodes on its final float32 poses of every slot row, whose results are appended to the bytes read.  With a
        threshold set the variant takes the verified rows (int32 [n], 0: the row's sequence re-detected or pads the batch)
        as its last input, and g6d_instances_verify_update applies the verdicts to live, ids and misses after the body
        packed them; its dropped ids go before the verification rows."""
        nodes, update = self._verify_fn(st), self._verify.resets

        def fn(frames, cams, *args):
            if update:
                *args, verified = args
            outs = body(frames, cams, *args)
            checked = nodes(frames, cams, outs[1], True)                      # [n, 10]: judge output, lost, window
            parts = [outs[0]]
            if update:
                lost = checked[:, 5].to(torch.int32).contiguous()
                live, ids, misses = outs[3:6]
                parts.append(ops.instances_verify_update(lost, verified, self.max_misses, live, ids, misses).view(torch.uint8))
            return (torch.cat(parts + [checked.reshape(-1).view(torch.uint8)]), *outs[1:])
        return fn

    # -------------------------------------------------------------- one step
    def step(self, frames, Ks, out=None, sequences=None, boxes=None):
        """frames: S uint8 [h,w,3] (of one size or several, row f13; or device frames, row f14, as Tracker.step takes them);
        Ks: [S,3,3]; out: drawing destinations as Tracker.step takes them (a tracker made with draw= draws every live slot
        of a sequence on its frame, in slot order; without out= inter['drawn'] holds tracker-owned frames).  Returns (poses float32 [S,M,3,4], smoothed float64 [S,M,3,4],
        track_ids int64 [S,M] (-1: empty slot), inter): inter['refine_poses'] a list of [S,M,3,4] (entry 0 the starting
        poses, float64 on a re-detection step; a row whose chain is shorter repeats its final pose), 'bbox_pts' and
        'smoothed_pts' [S,M,8,2].  Empty slots' poses and points are NaN.  A re-detection step adds predict_instances'
        keys led by [S,M], 'det_slot' int64 [S,M] (the slot detection m went to, -1: discarded), 'spawned' bool [S,M]
        (the slots that started a track) and 'dropped' (the ids removed this step, ascending).

        On the per-sequence schedules (row f18) inter['detected'] (bool [n]) marks the sequences that re-detected; when
        any did, the re-detection keys cover every row, the others' filled with NaN, -1, False / 0 and zero crops, and
        refine_poses has max(cfg['refine_iter'], refine_iter) + 1 entries.  sequences: step only these sequences, with
        Tracker.step's contract (row f17): one frame, K and out= destination each, in any order; results in that order
        with inter['sequences']; the others are not computed and keep their state and out= buffers.

        boxes (row f19): re-detect from another detector's boxes instead of running the detector, one entry per stepped
        sequence (in sequences= order, else 0..S-1): the boxes Gen6DEstimator.predict_instances(boxes=) takes for a frame
        ([n, 4|5], n >= 0), or None for none.  The boxes' records go through the same association and refinement as a
        detection; the detector runs no kernel.  Lockstep: every entry must be an array (an empty one: no detections),
        and the step is a re-detection step that restarts the re-detection count.  Per-sequence schedules: exactly the
        sequences given an array re-detect, and each counts as re-detected; a due sequence given None is not detected
        and stays due (detecting()).  So redetect_every=None with boxes on the first step never runs the detector.

        A tracker made with verify_every (row f21) adds inter['verify'] to the steps that verify: verify_poses' keys [S,M]
        on the step's final poses (empty slots and sequences that re-detected on the step: lost False, NaN), and with a
        threshold 'dropped', the ids the verdicts removed.  poses, smoothed and track_ids are the step's own; a dropped
        track's id is -1 from the next step on, and the sequences with a lost track re-detect on their next step."""
        return self._step(frames, Ks, out, sequences, boxes)[0]

    def _step(self, frames, Ks, out=None, sequences=None, boxes=None):
        """One step -> the decoded results of every object, in object order."""
        self._check()
        if self.schedule != 'lockstep':
            return self._step_sequences(frames, Ks, out, sequences, boxes)
        if sequences is not None:
            raise ValueError("step: sequences= needs schedule='per_sequence' or 'staggered'; a lockstep tracker's "
                             're-detection schedule is tracker-wide')
        est, S = self.est, self.S
        if len(frames) != S or len(Ks) != S:
            raise ValueError(f'step: this tracker follows {S} sequences, got {len(frames)} frames and {len(Ks)} Ks')
        Ks = np.stack([np.asarray(k) for k in Ks], 0)
        if Ks.shape != (S, 3, 3):
            raise ValueError(f'step: Ks must be [{S},3,3], got {Ks.shape}')
        table = None
        if boxes is not None:
            table, has = self._boxes(boxes, S)
            if not has.all():
                raise ValueError(f'step: a lockstep step with boxes re-detects every sequence; sequences '
                                 f'{np.flatnonzero(~has).tolist()} have None (pass an empty [0, 4] array for no detections)')
        detecting = table is not None or self._detecting()
        res = self._run(frames, Ks, out, 'detect' if detecting else 'refine', boxes=table)
        self._pending = False
        self._since = 1 if detecting else self._since + 1
        self._mark_lost(res, np.arange(S))
        return res

    def _boxes(self, boxes, n):
        """A step's boxes for n stepped sequences -> (boxes.Table of their maps, has bool [n])."""
        return B.for_sequences(boxes, n, 'step', self.est.detector.device)

    def _run(self, frames, Ks, out, kind, part=None, det_seq=None, boxes=None):
        """One step's graph and read -> decoded results.  kind: 'detect', 'refine' or 'mixed'; part: a partial step (row
        f17/f18) over its compact batch; det_seq: bool over the batch's sequences, those that re-detect (kind 'mixed');
        boxes: a boxes.Table of the batch's maps, the detection of a 'detect' or 'mixed' step (row f19).  The step
        verifies (row f21) when the schedule says so; its results then hold inter['verify']."""
        est = self.est
        S, stepped, refining, check = self._verify_plan(kind, part, det_seq)
        F = est.cfg['refine_iter']
        if kind != 'refine' and F < 1:
            raise ValueError("instance tracking needs cfg['refine_iter'] >= 1 (a re-detection step smooths float32 poses)")
        imgs = fr.as_frames(frames, 'step', est.detector)
        plan = fr.FramePlan(fr.size_pattern(imgs))
        if plan.mixed:
            fr.check_frames(imgs, Ks, 'step')
        stt, x = self._tables(), self._state
        drawer = self._drawer if part is None or self._drawer is None else self._drawer.for_sequences(part.b)
        draw, dt, drawn, named = draw_inputs(drawer, est.detector, plan, out, None if part is None else part.a)
        dev = est.detector.device
        up = lambda a, dt_: torch.from_numpy(np.ascontiguousarray(a, dt_)).to(dev)
        det_rows, extra, D, vin = None, [], S, []
        dbox = tail = None
        if boxes is not None and kind != 'refine':
            dbox = B.Detect(self.M, self.K, boxes.n_maps, boxes.N, B.inv_box_size(est.cfg['ref_resolution']))
            tail = [boxes.upload(est.detector)]
        if kind == 'mixed':
            seq, blocks, det_rows, D, key = plan_mixed(det_seq, plan)
            extra = [up(seq, np.int64), up(det_rows, np.int32)]
            base, fn = mixed_name(S, key), self._body(stt, 'mixed', S, D, blocks, draw, dbox)
        elif part is None and not check:
            base = kind
            fn = self._detect_fn(stt, draw, boxes=dbox) if kind == 'detect' else self._refine_fn(stt, draw)
        else:
            base, fn = kind, self._body(stt, kind, S, draw=draw, boxes=dbox)
        if check:                                  # the verifying variant takes and returns the whole slot state
            base, fn = V.graph_name(base, self._verify.key), self._verifying(fn, stt)
            if self._verify.resets:
                vin = [up(np.tile(refining, self.M * self.K), np.int32)]
        if dbox is not None:
            base, fn = B.graph_name(base, boxes.N), dbox.bind(fn)
        if part is not None:
            base = part.name(base)
            fn = _compact_state_fn(fn)
            extra = part.graph_inputs(dev) + extra
        with torch.no_grad():
            name, fn, fin = fr.stage(est.detector, named(base), fn, imgs, plan)
            cams = est.detector._to_dev(glue.cameras(Ks))
            if part is None and kind == 'refine' and not check:
                outs = self.stages.run(name, fn, fin + [cams, x['prev'], x['park'], x['live'], x['ids'], x['ring'], x['count']] + dt)
                buf, poses, ring, count = outs
            else:
                outs = self.stages.run(name, fn, fin + [cams, x['prev'], x['park'], x['live'], x['ids'], x['misses'], self._next_id,
                                                        x['ring'], x['count']] + extra + dt + vin + (tail or []))
                buf, poses, park, live, ids, misses, next_id, ring, count = outs
                for k, v in (('park', park), ('live', live), ('ids', ids), ('misses', misses)):
                    x[k].copy_(v)
                self._next_id.copy_(next_id)
            x['prev'].copy_(poses)
            x['ring'].copy_(ring)
            x['count'].copy_(count)
            host = est.detector._to_host(buf)                        # the step's one synchronising read
        if check:
            host, checked, dropped = self._split_verify(host, self.M * self.K * S)
        res = self._decode(host, kind != 'refine', S, det_rows, D)
        if drawn is not None:
            for r in res:
                r[3]['drawn'] = drawn
        if check:
            self._verify_results(res, checked, dropped, refining, S)
        self._verify_done(stepped, refining, check)
        return res

    def _verify_plan(self, kind, part=None, det_seq=None):
        """A step's verification plan (row f21) -> (S: the batch's sequences, stepped: the real ones' tracker indices,
        refining bool [S]: the batch rows that do not re-detect, padding excluded, check: the step verifies)."""
        S = self.S if part is None else part.b
        stepped = np.arange(self.S) if part is None else part.seq[:part.a]
        refining = np.full(S, kind == 'refine') if det_seq is None else ~np.asarray(det_seq, bool)
        refining[len(stepped):] = False
        return S, stepped, refining, self._verify.due_rows(self._vsince[stepped], refining[:len(stepped)])

    def _verify_done(self, stepped, refining, check):
        """The verification counts after the step: re-detected sequences restart, the others count the step, and a
        verifying step restarts every stepped sequence."""
        V.Schedule.advance(self._vsince, stepped, ~refining[:len(stepped)], check)

    def _split_verify(self, host, n):
        """A verifying step's read -> (the step body's bytes, verify.decode's dict of its n slot rows, the update's dropped
        int64 [n] or None without a threshold)."""
        host, checked = V.split(host, n)
        dropped = None
        if self._verify.resets:
            host, dropped = host[:len(host) - n * 8], host[len(host) - n * 8:].view(np.int64)
        return host, checked, dropped

    def _verify_results(self, res, checked, dropped, refining, S):
        """inter['verify'] of every object: verify_poses' keys [S, M] in the step's row order, rows of empty slots and of
        sequences that did not refine (re-detected, or padding) lost False and NaN; 'dropped' (with a threshold) the ids
        the update removed, ascending."""
        M, K = self.M, self.K
        for o, (_, _, ids, inter) in enumerate(res):
            skip = (ids < 0) | ~refining[:, None]
            v = {}
            for k, a in checked.items():
                a = instances.frame_major(a.reshape(M, K, S, *a.shape[1:])[:, o].reshape(M * S, *a.shape[1:]), M, S)
                a[skip] = False if a.dtype == bool else np.nan
                v[k] = a
            if dropped is not None:
                v['dropped'] = sorted(int(i) for i in dropped.reshape(M, K, S)[:, o].reshape(-1) if i >= 0)
            inter['verify'] = v

    def _mark_lost(self, res, seqs):
        """After a verifying step with a threshold set: every stepped sequence (seqs, the leading rows of the step's
        batch) with a slot judged lost re-detects on its next step, as redetect([s]) does; a lockstep tracker re-detects
        together, as redetect() does."""
        if not self._verify.resets or 'verify' not in res[0][3]:
            return
        lost = np.any([r[3]['verify']['lost'][:len(seqs)].any(1) for r in res], 0)
        if lost.any():
            self.redetect(None if self.schedule == 'lockstep' else seqs[lost])

    def _step_sequences(self, frames, Ks, out, sequences, boxes=None):
        """A step on a per-sequence schedule (row f18): the stepped sequences' plan, one graph, their counters.  boxes (row
        f19): per stepped sequence an array or None; the sequences with an array re-detect, from them."""
        S, sch = self.S, self._schedule
        part = None
        if sequences is not None:
            part = PartialStep(S, self.M * self.K, sequences, sch.due(), np.ones(S, bool), 1)
            part.check(frames, Ks, out)
            if out is not None and self._drawer is None:
                raise ValueError('step: out= names drawing destinations; create the tracker with draw=')
            frames, Ks, out = part.compact(frames), part.compact(Ks), part.compact_out(out)
            seqs, n_real = part.seq, part.a
            if boxes is not None:
                B.check_len(boxes, n_real, 'step', 'stepped sequence')
                boxes = part.compact(list(boxes))[:n_real] + [None] * (part.b - n_real)       # padding rows never detect
        else:
            if len(frames) != S or len(Ks) != S:
                raise ValueError(f'step: this tracker follows {S} sequences, got {len(frames)} frames and {len(Ks)} Ks')
            seqs, n_real = np.arange(S), S
            if boxes is not None:
                B.check_len(boxes, S, 'step', 'stepped sequence')
        Ks = np.stack([np.asarray(k) for k in Ks], 0)
        if Ks.shape != (len(seqs), 3, 3):
            raise ValueError(f'step: Ks must be [{len(seqs)},3,3], got {Ks.shape}')
        table = hit = None
        if boxes is not None:
            table, hit = self._boxes(boxes, len(seqs))
        det_seq, kind = sch.plan(seqs, n_real, hit)
        res = self._run(frames, Ks, out, kind, None if part is None or part.lockstep else part, det_seq, table)
        sch.advance(seqs[:n_real], det_seq[:n_real])
        self._mark_lost(res, seqs[:n_real])
        for r in res:
            r[3]['detected'] = det_seq.copy()
        if part is None:
            return res
        return [_reorder(r, part) for r in res]

    def _decode(self, host, detecting, S=None, det_rows=None, D=None):
        """det_rows: a mixed step's detection row of each sequence ([S], -1: not detecting) in its batch of D rows, whose
        parts are spread over the S rows (the others filled); None: every sequence detected at its own row."""
        est, M, K, num = self.est, self.M, self.K, self.num
        S = S or self.S
        D = S if D is None else D
        n = M * K * S
        n_chain = (max(est.cfg['refine_iter'], self.refine_iter) if detecting else self.refine_iter) + 1
        res = est.cfg['ref_resolution']
        rd = instances.Unpacker(host, M * K * D * res * res * 3 if detecting else 0)
        chain = rd.take(n_chain * n * 12).reshape(n_chain, n, 12)
        smoothed, avg = rd.take(n * 12).reshape(n, 12), rd.take(n * 16).reshape(n, 16)
        ring_h, count_h = rd.take(n * num * 16).reshape(n, num, 8, 2).astype(np.float32), rd.take(n).astype(np.int64)
        ids = rd.take(n)
        if detecting:
            nd = M * K * D
            det, sels = rd.take(nd * 4).reshape(nd, 4), self._take_selections(rd, D)
            valid, inst_count = rd.take(nd), rd.take(K * D).reshape(K, D)
            det_slot, spawned, dropped = rd.take(n), rd.take(n), rd.take(n)
            crops = rd.crops.reshape(nd, res, res, 3)
            if det_rows is not None:
                sp = lambda a, L, fill: _spread(a, L, D, det_rows, fill)
                det, valid, crops = sp(det, M * K, np.nan), sp(valid, M * K, 0), sp(crops, M * K, 0)
                inst_count = sp(inst_count.reshape(-1), K, 0).reshape(K, S)
                sels = [(sp(i, M, -1), sp(so.reshape(M * D, 2), M, np.nan).reshape(-1), sp(lg.reshape(M * D, -1), M, np.nan).reshape(-1))
                        for i, so, lg in sels]

        obj = lambda a, o: a.reshape(M, K, S, *a.shape[1:])[:, o].reshape(M * S, *a.shape[1:])      # object o, instance-major
        out = []
        for o in range(K):
            c = chain.reshape(n_chain, M, K, S, 12)[:, :, o].reshape(n_chain, M * S, 12)
            one = [obj(a, o) for a in (smoothed, avg, ring_h, count_h, ids)]
            det_parts = None
            if detecting:
                det_parts = [obj(det, o), *sels[o], obj(valid, o), inst_count[o], obj(crops, o),
                             *(obj(a, o) for a in (det_slot, spawned, dropped))]
            out.append(self._decode_object(c, *one, det_parts, o, S))
        return out

    def _decode_object(self, chain, smoothed, avg, ring_h, count_h, ids, det_parts, o, S=None):
        """One object's instance-major rows (row m*S + s) -> (poses, smoothed, track_ids, inter) as step() returns them."""
        S, M = S or self.S, self.M
        n = M * S
        ids = instances.frame_major(ids.astype(np.int64), M, S)
        empty = ids < 0
        fm = lambda a: instances.frame_major(a, M, S)

        def nan(a):
            a[empty] = np.nan
            return a
        first = fm(chain[0].reshape(n, 3, 4))
        detecting = det_parts is not None
        inter = {'refine_poses': [nan(first if detecting else first.astype(np.float32))] +
                                 [nan(fm(c.reshape(n, 3, 4)).astype(np.float32)) for c in chain[1:]],
                 'bbox_pts': nan(fm(ring_h[np.arange(n), count_h - 1])), 'smoothed_pts': nan(fm(avg.reshape(n, 8, 2)))}
        if detecting:
            det, idx, sel_out, logits, valid, inst_count, crops, det_slot, spawned, dropped = det_parts
            _, det_inter = instances.inter_of(chain[:1], det, idx, sel_out, logits, valid, inst_count, crops, M, S)
            det_inter.pop('refine_poses')
            inter.update(det_inter)
            inter['det_slot'] = fm(det_slot.astype(np.int64))
            inter['spawned'] = fm(spawned.astype(bool))
            inter['dropped'] = sorted(int(i) for i in dropped if i >= 0)
        return inter['refine_poses'][-1], nan(fm(smoothed.reshape(n, 3, 4))), ids, inter


def _spread(a, L, D, det_rows, fill):
    """Rows l*D + j of a detection batch -> rows l*S + s of the S sequences (j = det_rows[s]); rows of sequences that did
    not detect (det_rows -1) are `fill`."""
    S = len(det_rows)
    a = a.reshape(L, D, *a.shape[1:])
    out = np.full((L, S) + a.shape[2:], fill, a.dtype)
    s = np.flatnonzero(det_rows >= 0)
    out[:, s] = a[:, det_rows[s]]
    return out.reshape(L * S, *a.shape[2:])


def _compact_state_fn(fn):
    """A per-sequence step body fn(frames, cams, prev, park, live, ids, misses, next_id, ring, count, *rest) of a compact
    batch -> the partial step's body g(frames, cams, <the same state>, gather, scatter, *rest) on the tracker's whole slot
    state (PartialStep's rows over the M*K slot groups): gather the compact rows, run fn, copy the real rows back."""
    def g(frames, cams, prev, park, live, ids, misses, next_id, ring, count, gather, scatter, *rest):
        state = (prev, park, live, ids, misses, ring, count)
        p, pk, lv, i, ms, ring_c, count_c = _gather_rows(state, gather)
        outs = fn(frames, cams, p, pk, lv, i, ms, next_id, ring_c, count_c, *rest)
        buf, next_id = outs[0], outs[6]
        new = outs[1:6] + outs[7:9]
        return (buf, *[_scatter_rows(t, c, scatter) for t, c in zip(state[:5], new[:5])], next_id,
                *[_scatter_rows(t, c, scatter) for t, c in zip(state[5:], new[5:])])
    return g


def _reorder(res, part):
    """One object's results over a partial step's compact rows -> the listed sequences', in the caller's order, through
    PartialStep.results; 'dropped' (ids, not rows) passes through."""
    poses, smoothed, ids, inter = res
    inter = dict(inter)
    dropped = inter.pop('dropped', None)
    verify_dropped = inter['verify'].pop('dropped', None) if 'verify' in inter else None
    poses, smoothed, inter = part.results(poses, smoothed, inter)
    if dropped is not None:
        inter['dropped'] = dropped
    if verify_dropped is not None:
        inter['verify']['dropped'] = verify_dropped
    return poses, smoothed, ids[part.pos], inter


class ObjectInstanceTracker(InstanceTracker):
    """Every instance of every object of an ObjectSet tracked through S sequences in lockstep; see
    ObjectSet.instance_tracker().  Slot group g = m*K + o is instance slot m of object o; row g*S + s is that slot on
    sequence s.  reset(sequences) drops those sequences' tracks for every object."""

    def __init__(self, objs, num_sequences, max_instances=4, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1,
                 min_score=None, nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5, bboxes=None, draw=None,
                 draw_colors=None, schedule='lockstep', verify_every=None, lost_score=None, lost_gate=None):
        key = check_args(num_sequences, max_instances, refine_iter, redetect_every, gate, max_misses, min_score, nms_iou,
                         peak_radius, smooth_num, smooth_std, schedule)
        verify = V.Schedule(verify_every, lost_score, lost_gate)
        objs._check()
        boxes = object_bboxes(objs, bboxes)
        self.objs, self.names, self.bboxes = objs, objs.names, np.ascontiguousarray(np.stack(boxes, 0))
        self._membership = objs.membership
        self._setup(objs.est, key, boxes, num_sequences, refine_iter, redetect_every, gate, max_misses, smooth_num, smooth_std,
                    draw, dr.object_colors(self.names, draw_colors), schedule, verify)
        centers = np.stack([np.asarray(ob.ref_info['center'], np.float64).reshape(3) for ob in objs._objects.values()], 0)
        self._dev['centers'] = torch.from_numpy(np.ascontiguousarray(centers)).to(self.est.detector.device)

    def _check(self):
        if self.objs.membership != self._membership:
            raise RuntimeError('this instance tracker is stale: objects were added to or removed from the set since it was '
                               'created; create a new one with objs.instance_tracker()')
        self.objs._check()

    def _tables(self):
        return None

    def _groups(self, st):
        objs = list(self.objs._objects.values())
        return [ob.tables['views'] for ob in objs] * self.M, objs[0].tables['tables']['ref_num']

    def _detection(self, st, boxes=None):
        detect, extra = (boxes, boxes.extra) if boxes is not None else self.objs._peaks_detect_fn(*self.key)
        initial = self.objs._initial_poses_device_fn(detect)

        def fn(frames, cams):
            init, det, sels, crop = initial(frames, cams)
            return (init, det, crop, [t for sel in sels for t in sel], *extra)
        return fn

    def _associate(self):
        centers, est = self._dev['centers'], self.est
        return lambda det, valid, init, cams, *state: ops.instances_associate_objects(
            det, valid, init, cams, centers, float(est.cfg['ref_resolution']), self.gate, self.max_misses, est.cfg['refine_iter'],
            self.refine_iter, *state)

    def _boxes(self, boxes, n):
        return B.for_sequences(boxes, n, 'step', self.est.detector.device, self.names)

    def _verify_fn(self, st):
        return self.objs._verify_fn(self._verify.key, self.M)

    def _take_selections(self, rd, S):
        M, K = self.M, self.K
        n_sel = [len(ob.ref_info['poses']) for ob in self.objs._objects.values()]
        slots = [(rd.take(S), rd.take(S * 2), rd.take(S * n_sel[g % K])) for g in range(M * K)]
        return [tuple(np.concatenate([slots[m * K + o][i] for m in range(M)]) for i in range(3)) for o in range(K)]

    def step(self, frames, Ks, out=None, sequences=None, boxes=None):
        """frames: S uint8 [h,w,3] (of one size or several, row f13; or device frames, row f14); Ks: [S,3,3] (shared by all
        objects); out: drawing destinations as InstanceTracker.step takes them, every live slot of every object drawn.  Returns {name: (poses float32
        [S,M,3,4], smoothed float64 [S,M,3,4], track_ids int64 [S,M], inter)}: per object what InstanceTracker.step returns,
        'det_score' included on a re-detection step; 'dropped' lists that object's ids only.  Ids are unique over every
        object of the tracker.  sequences (per-sequence schedules, row f18): step only these, as InstanceTracker.step.
        boxes (row f19): as InstanceTracker.step takes them, each entry a dict {object name: boxes} (an object missing from
        it has no boxes on that frame) or None."""
        return dict(zip(self.names, self._step(frames, Ks, out, sequences, boxes)))
