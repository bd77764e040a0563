"""Video tracking (the reference's predict.py:47-70): a full prediction on the first frame, then `refine_iter`
refinements per frame starting from the previous frame's pose, and predict.py's temporal smoothing (the object's 3-D
box projected with every raw pose, an exponentially weighted average of the last `smooth_num` frames' corners, and a
PnP solve back to a pose).

With cfg['device_glue'] a tracking step for S sequences in lockstep is ONE captured graph -- the refinement chain
(csrc/glue.cu + the refiner) followed by the smoothing kernel (csrc/track.cu) -- and one synchronising read; the
previous poses and the corner histories stay on the device between steps.  Otherwise the host sequences the step
with predict_batch's host path and runs the smoothing through g6d_track_smooth_host (same code, on the CPU).

ObjectTracker (ObjectSet.tracker()) does the same for every object of an object set at once: one graph per step whose
glue and smoothing launches (the g6d_*_objects entry points) and refiner stage cover all K objects' K*S rows.  It is
Tracker's subclass: the state, the step driver (checks, partial steps, verification) and the decode of a step's read are
Tracker's, written for K object-major rows per sequence (K = 1 for Tracker); each class supplies its graph bodies, its
start() poses and its result shape.

reset(sequences) / start(poses, sequences) re-initialise or restart single sequences while the others keep tracking;
the step after them is the mixed step below, also one graph and one read.

step(..., sequences=[...]) steps a subset of the sequences and leaves the others untouched (the partial step below), so
streams at different frame rates, or that pause, share one tracker; S is then its capacity.

verify_every (row f20) makes every verify_every-th refine step of a sequence replay the verifying variant of the refine
graph (gen6d_b200/verify.py): the same body, then the detector on a window around each final pose, in the same read;
sequences judged lost are re-initialised as reset([s]) does.
"""
import copy

import numpy as np
import torch

from . import _lib
from . import draw as dr
from . import frames as fr
from . import glue
from . import ops
from . import verify as V
from .graphs import StageCache


# ------------------------------------------------------------------------------------------ smoothing inputs
def smoothing_weights(num, std):
    """predict.py:19 weighted_pts' weights, oldest frame first (the expression the reference evaluates)."""
    return np.ascontiguousarray(np.exp(-(np.arange(num) / std) ** 2)[::-1])


def bbox_from_points(pts):
    """utils/draw_utils.py pts_range_to_bbox_pts(max(pts), min(pts)): the 8 corners (float32, the reference's order).
    A box with zero extent along an axis (coplanar corners) is rejected: the smoothing's PnP solves the non-planar case
    only, where the reference would fall back to OpenCV's homography initialisation."""
    pts = np.asarray(pts)
    hi, lo = np.max(pts, 0), np.min(pts, 0)
    (maxx, maxy, maxz), (minx, miny, minz) = hi, lo
    box = np.asarray([[minx, miny, minz], [minx, maxy, minz], [maxx, maxy, minz], [maxx, miny, minz],
                      [minx, miny, maxz], [minx, maxy, maxz], [maxx, maxy, maxz], [maxx, miny, maxz]], np.float32)
    check_bbox(box)
    return box


def check_bbox(box):
    box = np.asarray(box, np.float32)
    if box.shape != (8, 3) or not np.isfinite(box).all():
        raise ValueError(f'bbox_3d must be 8 finite corners [8,3], got shape {box.shape}')
    ext = box.max(0) - box.min(0)
    if (ext <= 0).any():
        raise ValueError(f'bbox_3d has zero extent along an axis ({ext.tolist()}): its corners are coplanar, and the '
                         'smoothing solves the PnP for non-coplanar corners only')
    return np.ascontiguousarray(box)


def object_bbox(database):
    """The box predict.py smooths with: from the database's object point cloud (`object_point_cloud`, as on this
    package's SyntheticObjectDatabase and the reference's CustomDatabase), or, for a wrapped reference database, the
    reference's get_ref_point_cloud.  None when neither exists."""
    pc = getattr(database, 'object_point_cloud', None)
    if pc is None and hasattr(database, 'db'):          # database.ReferenceDatabaseAdapter
        pc = getattr(database.db, 'object_point_cloud', None)
        if pc is None:
            try:
                from dataset.database import get_ref_point_cloud   # reference package
                pc = get_ref_point_cloud(database.db)
            except (ImportError, NotImplementedError, AttributeError):
                pc = None
    return None if pc is None else bbox_from_points(pc)


def object_bboxes(objs, bboxes):
    """The box of every object of an ObjectSet, in set order: bboxes[name] (8 corners [8,3]) where given, else the box of
    the object's database point cloud."""
    bboxes = dict(bboxes or {})
    unknown = sorted(set(bboxes) - set(objs.names))
    if unknown:
        raise ValueError(f'bboxes names objects that are not in the set: {unknown} (objects: {objs.names})')
    boxes = []
    for name, ob in objs._objects.items():
        box = bboxes.get(name)
        if box is None:
            box = object_bbox(ob.ref.database)
            if box is None:
                raise ValueError(f'object {name!r}: its database has no object point cloud: pass bboxes[{name!r}] (the 8 '
                                 'corners of the object box)')
        boxes.append(check_bbox(box))
    return boxes


def host_smooth(poses, poses_are_f32, bbox, Ks, ring, count, weights):
    """g6d_track_smooth_host on numpy arrays: poses [S,3,4] / [S,12], Ks [S,3,3]; ring float32 [S,num,8,2] and count
    int32 [S] are updated in place.  Returns (smoothed float64 [S,3,4], averaged corners float64 [S,8,2])."""
    S = len(poses)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(S, 12))
    K = np.ascontiguousarray(np.asarray(Ks, np.float64).reshape(S, 9))
    box = np.ascontiguousarray(bbox, np.float32)
    w = np.ascontiguousarray(weights, np.float64)
    for a, dt in ((ring, np.float32), (count, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_smooth: ring / count must be contiguous {dt.__name__} arrays (updated in place)')
    smoothed, avg = np.zeros((S, 12), np.float64), np.zeros((S, 8, 2), np.float64)
    _lib.check(_lib.lib().g6d_track_smooth_host(p.ctypes.data, int(poses_are_f32), box.ctypes.data, K.ctypes.data,
                                                ring.ctypes.data, count.ctypes.data, ring.shape[1] if ring.ndim > 1 else 0,
                                                w.ctypes.data, S, smoothed.ctypes.data, avg.ctypes.data),
               'g6d_track_smooth_host')
    return smoothed.reshape(S, 3, 4), avg


def host_smooth_objects(poses, poses_are_f32, bboxes, Ks, ring, count, weights):
    """g6d_track_smooth_objects_host on numpy arrays: K objects through S sequences, rows object-major (row o*S + s):
    poses [K*S,3,4], bboxes [K,8,3], Ks [S,3,3]; ring float32 [K*S,num,8,2] and count int32 [K*S] are updated in place.
    Returns (smoothed float64 [K*S,3,4], averaged corners float64 [K*S,8,2])."""
    n, K, S = len(poses), len(bboxes), len(Ks)
    p = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(n, 12))
    K9 = np.ascontiguousarray(np.asarray(Ks, np.float64).reshape(S, 9))
    box = np.ascontiguousarray(bboxes, np.float32)
    w = np.ascontiguousarray(weights, np.float64)
    for a, dt in ((ring, np.float32), (count, np.int32)):
        if a.dtype != dt or not a.flags.c_contiguous:
            raise ValueError(f'host_smooth_objects: ring / count must be contiguous {dt.__name__} arrays (updated in place)')
    smoothed, avg = np.zeros((n, 12), np.float64), np.zeros((n, 8, 2), np.float64)
    _lib.check(_lib.lib().g6d_track_smooth_objects_host(p.ctypes.data, int(poses_are_f32), box.ctypes.data, K, S, K9.ctypes.data,
                                                        ring.ctypes.data, count.ctypes.data, ring.shape[1] if ring.ndim > 1 else 0,
                                                        w.ctypes.data, smoothed.ctypes.data, avg.ctypes.data),
               'g6d_track_smooth_objects_host')
    return smoothed.reshape(n, 3, 4), avg


# ------------------------------------------------------------------------------------------ the mixed step
# A step in which some sequences are re-initialised (a full prediction) and the others refine from their previous pose,
# or in which the rows' previous poses have different dtypes.  It is one captured graph: the re-initialised sequences'
# frames are gathered and run through detection, selection and the initial poses as a batch padded to a power of two
# (the bucket b, capped at S: the padding repeats a re-initialised sequence), the initial poses are scattered into a
# working array [K*(S+b),12] that holds the other rows' previous poses (per object S real rows, then b scratch rows), and
# max(cfg['refine_iter'], refine_iter) iterations refine the rows whose chain is still running, in ascending row order,
# through the row-indexed glue and ONE refiner stage per iteration.  Every shape depends on the bucket only, so every
# subset of a bucket replays one graph: an iteration in which every real row refines lists exactly the S real rows (the
# refiner stage of a plain refine step), and a shorter list is padded with scratch rows to a length fixed by the bucket;
# scratch rows hold copies of the bucket's initial poses and their results are dropped.
def _bucket(m, S):
    return 0 if m == 0 else min(S, 1 << (m - 1).bit_length())


def _iter_lengths(S, b, F, r):
    """Rows per object of each refinement iteration (F: the re-initialised rows' chain length, r: the others')."""
    return [S if (it < F and it < r) or it >= F else b for it in range(max(F, r))]


def _size_buckets(reinit, plan):
    """The re-initialised sequences of a step over frames of different sizes, bucketed per size (row f13) -> (gathered
    sequences [b], rows per size group [b_z], each re-initialised sequence's position in the gather [m]).  Per size group
    of g sequences with m_z of them re-initialised, b_z = _bucket(m_z, g): its re-initialised sequences in ascending order,
    padded by repeating the last; the blocks follow the groups' order."""
    seq, blocks, pick = [], [], np.zeros(len(reinit), np.int64)
    for _, _, idx, _ in plan.groups:
        mine = reinit[np.isin(reinit, idx)]
        bz = _bucket(len(mine), len(idx))
        pick[np.searchsorted(reinit, mine)] = len(seq) + np.arange(len(mine))
        seq += list(mine) + [mine[-1]] * (bz - len(mine)) if bz else []
        blocks.append(bz)
    return np.asarray(seq, np.int64), blocks, pick


def _mixed_inputs(S, K, pending, f32, F, r, device, plan=None):
    """Host side of a mixed step -> (re-initialised sequences [m], bucket, graph inputs: gathered sequences int64 [b], scatter
    rows int64 [K*b], first-iteration dtype flags uint8 [K*(S+b)], the iterations' row lists int32, object-major).
    plan: the FramePlan of frames of different sizes, whose buckets are per size (_size_buckets)."""
    reinit, others = np.flatnonzero(pending), np.flatnonzero(~pending)
    m = len(reinit)
    if plan is None or not plan.mixed:
        b = _bucket(m, S)
        seq = np.concatenate([reinit, np.full(b - m, reinit[-1] if m else 0)])
        tgt = np.concatenate([reinit, S + np.arange(m, b)])
    else:
        seq, _, pick = _size_buckets(reinit, plan)
        b = len(seq)
        tgt = S + np.arange(b)                                            # padding rows go to their scratch rows
        tgt[pick] = reinit
    n = S + b
    flags = np.zeros(n, np.uint8)
    flags[others] = f32[others]
    lists = []
    for it, L in enumerate(_iter_lengths(S, b, F, r)):
        if it < F and it < r:
            rows = np.arange(S)
        elif it < F:
            rows = np.concatenate([reinit, S + np.arange(b - m)])        # re-initialised rows only, padded to b
        else:
            rows = np.concatenate([others, S + np.arange(m)])            # the other rows only, padded to S
        assert len(rows) == L
        lists += [o * n + rows for o in range(K)]
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(device)
    tgt_k = np.concatenate([o * n + tgt for o in range(K)])
    inputs = [up(seq, np.int64), up(tgt_k, np.int64), up(np.tile(flags, K), np.uint8),
              up(np.concatenate(lists) if lists else np.zeros(0), np.int32)]
    return reinit, b, inputs


def _mixed_fn(K, S, b, F, r, initial, views, R, refine, smooth, blocks=None, draw=None):
    """The mixed step's graph body.  initial(frames, cams) -> (poses [K*b,12], crops, [tensors packed after the smoothing]);
    smooth(poses [K*S,12], poses_are_f32, Ks [S,9], ring, count) -> (smoothed, averaged corners).  blocks: the gathered
    rows per size group of frames of different sizes (_size_buckets), detected per size.  draw(frames, raw, raw_f32,
    smoothed, Ks, table): the draw node (row f16), run after the smoothing when the body is given a destination table."""
    n, lens = S + b, _iter_lengths(S, b, F, r)

    def fn(frames, cams, prev, ring, count, seq, tgt, flags0, lists, *dt):
        if b:
            gf, gc = frames.index_select(0, seq), cams.index_select(0, seq)
            if blocks is None:
                init, crop, extras = initial(gf, gc)
            else:
                with fr.gathered(frames, gf, seq, blocks):
                    init, crop, extras = initial(gf, gc)
            frames_x, cams_x = torch.cat([frames, gf], 0), torch.cat([cams, gc], 0)
            work = torch.cat([prev.view(K, S, 12), init.view(K, b, 12)], 1).reshape(K * n, 12)
            work.index_copy_(0, tgt, init)
        else:
            frames_x, cams_x, work, extras = frames, cams, prev.clone(), []
        real = lambda: work.view(K, n, 12)[:, :S].reshape(K * S, 12).clone()
        ones = torch.ones_like(flags0)
        chain, off = [real()], 0
        for it, L in enumerate(lens):
            if L:
                idx = lists[off:off + K * L]
                off += K * L
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_rows(views, R, n, cams_x, frames_x, work, idx,
                                                                                                  flags0 if it == 0 else ones)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)            # one refiner stage over the listed rows
                ops.glue_apply_refinements_rows(views, n, que_pose, que_K, rect, out, idx, work)
            chain.append(real())
        poses = chain[-1]
        Ks = cams[:, :9].contiguous()
        smoothed, avg = smooth(poses, True, Ks, ring, count)
        if dt:
            draw(frames, poses, True, smoothed, Ks, dt[0])
        packed = torch.cat([t.reshape(-1).to(torch.float64) for t in [torch.stack(chain, 0), smoothed, avg, ring, count] + extras])
        return (torch.cat([packed.view(torch.uint8), crop.reshape(-1)]) if b else packed.view(torch.uint8)), poses, ring, count
    return fn


def draw_inputs(drawer, module, plan, out, real=None):
    """A step's drawing (row f16) -> (draw hook for the graph body or None, [destination table] graph inputs, inter['drawn']
    or None, graph name map).  The destinations are checked here, before anything is enqueued.  real: the leading
    sequences of a compact batch that out= covers (a partial step, row f17; the others are padding)."""
    if drawer is None:
        if out is not None:
            raise ValueError('step: out= names drawing destinations; create the tracker with draw=')
        return None, [], None, (lambda n: n)
    table, drawn = drawer.destinations(module, plan, out, real)
    return (lambda *a: drawer.node(module, plan, *a)), [table], drawn, drawer.name


def _sequences(S, sequences):
    """Validated sequence indices, in the caller's order (start() pairs poses[i] with sequences[i])."""
    seqs = [int(s) for s in sequences]
    if len(set(seqs)) != len(seqs):
        raise ValueError(f'sequences {seqs} lists a sequence twice')
    bad = [s for s in seqs if not 0 <= s < S]
    if bad:
        raise ValueError(f'sequences {bad} are outside [0, {S})')
    return np.asarray(seqs, np.int64)


def _step_kind(pending, f32, F):
    """'full', 'refine' or 'mixed': the graph a step over sequences with these pending and float32 flags replays (F:
    cfg['refine_iter'])."""
    if pending.all():
        return 'full'
    if not pending.any() and (f32.all() or not f32.any()):
        return 'refine'
    if pending.any() and F < 1:
        raise ValueError("re-initialising some sequences while others track needs cfg['refine_iter'] >= 1 (the step "
                         'smooths float32 poses)')
    return 'mixed'


# ------------------------------------------------------------------------------------------ the partial step
# A step over a subset of the sequences (row f17): the a listed sequences, sorted and padded to b = _bucket(a, S) by
# repeating the last, run the unchanged step body of a b-sequence tracker on compact copies of their state rows, gathered
# inside the graph; only the a real rows are copied back.  The gather and scatter rows are graph inputs, so every list of
# one bucket (and step kind, size pattern and drawing) replays one graph.
class PartialStep:
    """The host plan of a partial step.  sequences: the caller's list (int64); seq: the compact batch's sequences [b],
    ascending, then padding; pos[i]: the compact row of sequences[i]; pending / f32: the compact rows' flags; kind: the
    step kind from them; gather int64 [K*b]: the tracker rows (object-major, o*S + s) of the compact rows o*b + j;
    scatter int64 [K*b]: where compact row o*b + j goes in [tracker rows; compact rows], its tracker row when real, its
    own copy (K*S + o*b + j) when padding; lockstep: every sequence is listed (the step is the lockstep step, reordered)."""

    def __init__(self, S, K, sequences, pending, f32, F):
        self.sequences = _sequences(S, sequences)
        if not len(self.sequences):
            raise ValueError('step: sequences lists no sequence; list at least one (or pass None for all)')
        order = np.argsort(self.sequences, kind='stable')
        self.S, self.K, self.a = S, K, len(order)
        self.lockstep = self.a == S
        self.b = S if self.lockstep else _bucket(self.a, S)
        self.order = np.concatenate([order, np.full(self.b - self.a, order[-1])])      # caller index of each compact row
        self.seq = self.sequences[self.order]
        self.pos = np.empty(self.a, np.int64)
        self.pos[order] = np.arange(self.a)
        self.pending, self.f32 = pending[self.seq].copy(), f32[self.seq].copy()
        self.kind = _step_kind(self.pending, self.f32, F)
        j = np.arange(self.b)
        self.gather = np.concatenate([o * S + self.seq for o in range(K)])
        self.scatter = np.concatenate([np.where(j < self.a, o * S + self.seq, K * S + o * self.b + j) for o in range(K)])

    def name(self, base):
        """The graph name of the compact batch's step `base` (a lockstep name): apart from every lockstep graph."""
        return (base, 'rows', self.b)

    def check(self, frames, Ks, out=None):
        """ValueError unless frames, Ks and every out= list hold one entry per listed sequence."""
        n = [len(frames), len(Ks)] + ([len(v) for v in out.values()] if isinstance(out, dict) else [])
        if any(m != self.a for m in n):
            raise ValueError(f'step: sequences lists {self.a} sequences; frames, Ks and every out= list need one entry each, '
                             f'got {len(frames)} frames, {len(Ks)} Ks' +
                             (f', out {({k: len(v) for k, v in out.items()})}' if isinstance(out, dict) else ''))

    def compact(self, items):
        """The caller's per-sequence entries in compact row order (padding repeats the last listed sequence's)."""
        return [items[i] for i in self.order]

    def compact_out(self, out):
        return None if out is None else {k: [v[i] for i in self.order[:self.a]] for k, v in out.items()}

    def graph_inputs(self, device):
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(device)
        return [up(self.gather), up(self.scatter)]

    def results(self, raw, smoothed, inter):
        """A step's results over the compact rows (ascending, padding last) -> the listed sequences' in the caller's order.
        A mixed step's 'reinit' becomes tracker-wide sequences (ascending) with their detection entries in that order."""
        pos = self.pos
        take = lambda v, idx: v[idx] if isinstance(v, np.ndarray) else [v[i] for i in idx]
        res = {}
        if 'reinit' in inter:
            r = np.asarray(inter['reinit'], np.int64)
            m = int((r < self.a).sum())                    # the real re-initialised rows come first (ascending)
        for k, v in inter.items():
            if k == 'reinit':
                res[k] = self.seq[r[:m]]
            elif k == 'drawn':
                res[k] = {kind: take(d, pos) for kind, d in v.items()}
            elif k == 'refine_poses':
                res[k] = [c[pos] for c in v]
            elif k == 'verify':
                res[k] = {kk: vv[pos] for kk, vv in v.items()}
            elif 'reinit' in inter and k not in ('bbox_pts', 'smoothed_pts'):
                res[k] = take(v, range(m))
            else:
                res[k] = take(v, pos)
        res['sequences'] = self.sequences.copy()
        return raw[pos], smoothed[pos], res


def _gather_rows(tensors, gather):
    """The compact rows (PartialStep.gather) of every state tensor."""
    return [t.index_select(0, gather) for t in tensors]


def _scatter_rows(t, c, scatter):
    """State tensor t with the compact rows c copied back (PartialStep.scatter: padding rows land in scratch copies,
    dropped)."""
    return torch.cat([t, c], 0).index_copy_(0, scatter, c)[:t.shape[0]]


def _compact_fn(fn, full):
    """A lockstep step body fn(frames, cams, [prev,] ring, count, *rest) of the compact batch -> the partial step's graph
    body g(frames, cams, prev, ring, count, gather, scatter, *rest) on the tracker's whole state: gather the compact rows,
    run fn, copy its real rows back (padding rows land in their scratch copies, dropped)."""
    def g(frames, cams, prev, ring, count, gather, scatter, *rest):
        sub = _gather_rows((ring, count) if full else (prev, ring, count), gather)
        buf, poses, ring_c, count_c = fn(frames, cams, *sub, *rest)
        put = lambda t, c: _scatter_rows(t, c, scatter)
        return buf, put(prev, poses), put(ring, ring_c), put(count, count_c)
    return g


# ------------------------------------------------------------------------------------------ the tracker
class Tracker:
    """S sequences tracked in lockstep (one frame each per step); see Gen6DEstimator.tracker().

    The state, the step driver and the decode of a step's read are written for K objects per sequence (K = 1 here), rows
    object-major (row o*S + s is object o on sequence s); ObjectTracker supplies an object set's graph bodies, start()
    poses and result shape through the hooks at the end of this class."""
    K = 1
    _host = True                     # steps may take the host path; the state stays on the host until a device step
    _verify = V.Schedule()           # no verification (row f20)

    def __init__(self, est, num_sequences, refine_iter=1, smooth_num=5, smooth_std=2.5, bbox_3d=None, draw=None,
                 draw_color=dr.DEFAULT_COLOR, verify_every=None, lost_score=None, lost_gate=None):
        kinds, draw_color = dr.parse_kinds(draw), dr.parse_color(draw_color)
        self._setup(est, num_sequences, refine_iter, smooth_num, smooth_std, verify_every, lost_score, lost_gate)
        if est.refiner is None:
            raise ValueError('tracking refines from the previous pose: the estimator needs a refiner')
        if bbox_3d is None:
            bbox_3d = object_bbox(est.refiner.ref_database)
            if bbox_3d is None:
                raise ValueError('the database has no object point cloud: pass bbox_3d (the 8 corners of the object box)')
        self.bbox = check_bbox(bbox_3d)
        self._gen = est._generation()
        self._dev = None                 # device copies of bbox / weights
        self.draw = kinds                # the kinds each step draws (row f16); None: no drawing
        self._drawer = dr.StepDrawer(kinds, [draw_color], self.bbox, [0], self.S, est.detector.device) if kinds else None
        self.reset()

    def _setup(self, est, num_sequences, refine_iter, smooth_num, smooth_std, verify_every, lost_score, lost_gate):
        """The arguments every tracker takes, checked, and the constants that do not depend on its objects."""
        if int(num_sequences) < 1:
            raise ValueError(f'num_sequences must be >= 1, got {num_sequences}')
        self._verify = V.Schedule(verify_every, lost_score, lost_gate)
        if int(refine_iter) < 1:
            raise ValueError(f'refine_iter must be >= 1, got {refine_iter}')
        if int(smooth_num) < 1:
            raise ValueError(f'smooth_num must be >= 1, got {smooth_num}')
        if not float(smooth_std) > 0:
            raise ValueError(f'smooth_std must be > 0, got {smooth_std}')
        self.est = est
        self.S, self.refine_iter = int(num_sequences), int(refine_iter)
        self.num, self.std = int(smooth_num), float(smooth_std)
        self.weights = smoothing_weights(self.num, self.std)
        self.stages = StageCache()       # this tracker's step graphs (they capture its device state)

    # -------------------------------------------------------------- state
    def reset(self, sequences=None):
        """The next step is a full prediction (detect -> select -> cfg['refine_iter'] refinements) for every object and
        sequence, and the smoothing histories restart.  sequences: only those sequences (every object on them) are
        re-initialised at the next step and restart their histories; the others keep tracking (that step is the mixed
        step)."""
        if sequences is None:
            n = self.K * self.S
            self._since = np.zeros(self.S, np.int64)  # refine steps since the last verification (row f20)
            self._prev = None                        # float64 previous poses ([K*S,12] on the device, [S,3,4] on the host)
            self._pending = np.ones(self.S, bool)    # a full prediction at the next step
            self._f32 = np.ones(self.S, bool)        # each sequence's previous poses hold float32 values
            self._ring = np.zeros((n, self.num, 8, 2), np.float32)
            self._count = np.zeros(n, np.int32)
            if not self._host:
                self._to(True)
            return
        seqs = _sequences(self.S, sequences)
        self._pending[seqs] = True
        self._restart(seqs)

    def _rows(self, seqs):
        """The state rows of sequences `seqs`, every object's (object-major), as an index into the state arrays."""
        rows = np.concatenate([o * self.S + seqs for o in range(self.K)])
        return rows if isinstance(self._ring, np.ndarray) else torch.from_numpy(rows).to(self._ring.device)

    def _restart(self, seqs):
        """Restart the smoothing of `seqs`: count 0 and a zero ring, the bytes of a fresh tracker's history; and their
        verification counts."""
        self._since[seqs] = 0
        if len(seqs):
            rows = self._rows(seqs)
            self._ring[rows] = 0
            self._count[rows] = 0

    def start(self, poses, sequences=None):
        """Begin (or restart) every sequence from known poses [S,3,4]: the next step refines from them, and the
        smoothing histories restart.  sequences: poses [len(sequences),3,4] for those sequences only; the others are
        unaffected.  A float32 array marks its poses as float32 values (as after a refinement), any other dtype float64."""
        seqs, p64, f32 = self._start_poses(poses, sequences)
        if sequences is None:
            self.reset()
        else:
            self._restart(seqs)
        if self._prev is None:
            self._prev = np.zeros((self.S, 3, 4)) if isinstance(self._ring, np.ndarray) else \
                torch.zeros(self.K * self.S, 12, dtype=torch.float64, device=self._ring.device)
        rows = self._rows(seqs)
        if isinstance(self._prev, np.ndarray):
            self._prev[rows] = p64.reshape(-1, 3, 4)
        else:
            self._prev[rows] = torch.from_numpy(p64).to(self._prev.device)
        self._pending[seqs] = False
        self._f32[seqs] = f32

    def _device_path(self):
        return not self._host or (bool(self.est.cfg['device_glue']) and self.est._glue_possible())

    def _to(self, device):
        """Move the previous poses and the histories to the device (torch tensors) or the host (numpy)."""
        if device:
            if not isinstance(self._ring, torch.Tensor):
                dev = self.est.detector.device
                self._ring, self._count = torch.from_numpy(self._ring).to(dev), torch.from_numpy(self._count).to(dev)
                if self._prev is not None:
                    self._prev = torch.from_numpy(np.asarray(self._prev, np.float64).reshape(self.S, 12)).to(dev)
        elif isinstance(self._ring, torch.Tensor):
            self._ring, self._count = self._ring.cpu().numpy(), self._count.cpu().numpy()
            if self._prev is not None:
                self._prev = self._prev.cpu().numpy().reshape(self.S, 3, 4)

    def _kind(self):
        """'full', 'refine' or 'mixed': the graph the next step replays."""
        return _step_kind(self._pending, self._f32, self.est.cfg['refine_iter'])

    def _partial(self, frames, Ks, out, sequences):
        """The plan of a step over `sequences` (row f17), its arguments checked before anything is enqueued."""
        part = PartialStep(self.S, self.K, sequences, self._pending, self._f32, self.est.cfg['refine_iter'])
        part.check(frames, Ks, out)
        if out is not None and self._drawer is None:
            raise ValueError('step: out= names drawing destinations; create the tracker with draw=')
        return part

    # -------------------------------------------------------------- one step
    def step(self, frames, Ks, out=None, sequences=None):
        """frames: S uint8 [h,w,3] (of different sizes on the device path, row f13; or, on that path, device frames with
        predict_batch's rules, row f14: CUDA RGB tensors and frames.NV12 surfaces, ready on the current stream and free to
        reuse when step returns); Ks: [S,3,3].  Returns (raw poses float32 [S,3,4], smoothed poses float64
        [S,3,4], inter): inter['refine_poses'] is this step's chain, inter['bbox_pts'] the projected box corners
        [S,8,2], inter['smoothed_pts'] their weighted average [S,8,2]; a full-prediction step adds the detection and
        selection entries of predict_batch.  A mixed step (some sequences re-initialised by reset(sequences), or previous
        poses of different dtypes) adds inter['reinit'] (the re-initialised sequences, ascending) with the detection and
        selection entries of those sequences in that order, and its chain has 1 + max(cfg['refine_iter'], refine_iter)
        entries [S,3,4]: entry 0 the starting poses (float64), a row whose chain is shorter repeating its final pose.

        A tracker made with draw= (row f16) draws predict.py's box into every frame inside the step's graph, as its last
        node: inter['drawn'] = {kind: S CUDA uint8 [h, w, 3] views of tracker-owned buffers at each frame's working size,
        overwritten by the next step}.  out={kind: S destinations} (CUDA uint8 RGB tensors of the working size with any
        row pitch, or frames.NV12 of an even working size) writes into the caller's buffers instead; they are written on
        the current stream.

        sequences (row f17): step only these sequences (distinct, in any order, at least one); frames, Ks and out's lists
        then hold one entry per listed sequence in that order, and every result (poses [n,3,4], each inter array, the
        drawn frames) comes back in that order, with inter['sequences'] echoing the list and a mixed step's
        inter['reinit'] holding tracker-wide sequences.  Each listed sequence takes exactly the step it would take in
        lockstep (a full prediction if pending, else refinement from its start or previous pose, then the smoothing over
        its own history); the others are untouched: no computation, their state and pending flags kept as they are.  The
        listed sequences run as a compact batch of _bucket(n, S) sequences (the last repeated as padding), one captured
        graph per bucket, step kind, size pattern and drawing, so results equal those of a tracker of that many
        sequences.  Listing every sequence is the lockstep step.

        A tracker made with verify_every (row f20) adds inter['verify'] to the refine steps that verify: verify_poses' keys
        on the step's final poses, in the step's row order; the sequences it judges lost are pending afterwards."""
        return self._results(self._step(frames, Ks, out, sequences))

    def _step(self, frames, Ks, out, sequences):
        """step() -> [(raw, smoothed, inter)] per object."""
        self._check()
        part = None
        if sequences is not None:
            part = self._partial(frames, Ks, out, sequences)
            frames, Ks, out = part.compact(frames), part.compact(Ks), part.compact_out(out)
            if part.lockstep:
                return [part.results(*r) for r in self._step(frames, Ks, out, None)]
        elif len(frames) != self.S or len(Ks) != self.S:
            raise ValueError(f'step: this tracker follows {self.S} sequences, got {len(frames)} frames and {len(Ks)} Ks')
        if out is not None and self._drawer is None:
            raise ValueError('step: out= names drawing destinations; create the tracker with draw=')
        S = self.S if part is None else part.b
        Ks = np.stack([np.asarray(K) for K in Ks], 0)
        if Ks.shape != (S, 3, 3):
            raise ValueError(f'step: Ks must be [{S},3,3], got {Ks.shape}')
        kind = self._kind() if part is None else part.kind
        device = self._device_path()
        if self._drawer is not None and not device:
            raise ValueError("drawing (draw=) runs inside the device pipeline's step graph only (cfg['device_glue'] on, "
                             "cfg['host_warps'] off)")
        if self._verify.every is not None and not device:
            raise ValueError("verification (verify_every=) runs inside the device pipeline's step graph only "
                             "(cfg['device_glue'] on, cfg['host_warps'] off)")
        host_path = "tracking with cfg['device_glue'] off or cfg['host_warps'] on"
        imgs = fr.as_frames(frames, 'step', self.est.detector, None if device else host_path)
        if not device:
            fr.require_one_size(frames, host_path)
        elif fr.is_mixed(imgs):
            fr.check_frames(imgs, Ks, 'step')
        stepped = np.arange(self.S) if part is None else part.seq[:part.a]
        pending, check = self._pending[stepped].copy(), self._verify.due(kind, self._since[stepped])
        if part is None:
            res = self._step_device(imgs, Ks, kind, out, check=check) if device else [self._step_host(frames, Ks, kind)]
            self._pending[:] = False
        else:
            res = self._step_device(imgs, Ks, kind, out, part, check) if device else \
                [self._step_host_partial(frames, Ks, kind, part)]
            self._pending[part.seq] = False
            res = [part.results(*r) for r in res]
        self._verify.advance(self._since, stepped, pending, check)
        if check:                                          # a sequence is lost when any of its objects is
            lost = np.any([r[2]['verify']['lost'] for r in res], 0)
            lost = self._verify.lost_sequences(stepped if part is None else part.sequences, lost)
            if len(lost):
                self.reset(lost)
        return res

    def _step_host_partial(self, frames, Ks, kind, part):
        """A partial step on the host path: _step_host on a view of this tracker holding the listed sequences' rows only
        (ascending, no padding), whose state is copied back."""
        self._to(False)
        seqs, a = part.seq[:part.a], part.a
        sub = copy.copy(self)
        sub.S, sub._pending, sub._f32 = a, part.pending[:a].copy(), part.f32[:a].copy()
        sub._prev = None if self._prev is None else self._prev[seqs]
        sub._ring, sub._count = self._ring[seqs], self._count[seqs]
        res = sub._step_host(frames[:a], Ks[:a], kind)
        if self._prev is None:
            self._prev = np.zeros((self.S, 3, 4))
        self._prev[seqs], self._f32[seqs] = sub._prev, sub._f32
        self._ring[seqs], self._count[seqs] = sub._ring, sub._count
        return res

    def _step_host(self, frames, Ks, kind):
        est, S = self.est, self.S
        self._to(False)
        if kind == 'full':
            poses, inter = est.predict_batch(frames, list(Ks))
        elif kind == 'refine':
            dev_frames = est.detector.upload_frame([np.asarray(f) for f in frames])
            prev = self._prev.astype(np.float32) if self._f32[0] else self._prev
            poses, chain = est._refine_batch_host(dev_frames, list(Ks), prev, self.refine_iter)
            inter = {'refine_poses': chain}
        else:
            poses, inter = self._mixed_host(frames, Ks)
        poses = np.asarray(poses)
        smoothed, avg = host_smooth(poses, poses.dtype == np.float32, self.bbox, Ks, self._ring, self._count, self.weights)
        self._prev = np.asarray(poses, np.float64).reshape(S, 3, 4).copy()
        self._f32[:] = poses.dtype == np.float32
        inter['bbox_pts'] = self._ring[np.arange(S), self._count - 1].copy()
        inter['smoothed_pts'] = avg
        return poses, smoothed, inter

    def _mixed_host(self, frames, Ks):
        """The mixed step on the host: predict_batch on the re-initialised frames, _refine_batch_host on the others (one
        call per dtype of their previous poses)."""
        est, S, F, r = self.est, self.S, self.est.cfg['refine_iter'], self.refine_iter
        reinit, others = np.flatnonzero(self._pending), np.flatnonzero(~self._pending)
        n_it = max(F, r)
        chain = np.zeros((n_it + 1, S, 3, 4))
        inter = {}
        if len(reinit):
            _, pb = est.predict_batch([frames[i] for i in reinit], list(Ks[reinit]))
            for k in range(n_it + 1):
                chain[k, reinit] = pb['refine_poses'][min(k, F)]
            inter.update({k: v for k, v in pb.items() if k != 'refine_poses'})
        for f32 in (True, False):
            rows = others[self._f32[others] == f32]
            if len(rows):
                dev_frames = est.detector.upload_frame([np.asarray(frames[i]) for i in rows])
                prev = self._prev[rows].astype(np.float32) if f32 else self._prev[rows]
                _, ch = est._refine_batch_host(dev_frames, list(Ks[rows]), prev, r)
                for k in range(n_it + 1):
                    chain[k, rows] = ch[min(k, r)]
        inter['reinit'] = reinit.astype(np.int64)
        inter['refine_poses'] = [chain[0]] + [c.astype(np.float32) for c in chain[1:]]
        return inter['refine_poses'][-1], inter


    def _step_device(self, imgs, Ks, kind, out=None, part=None, check=False):
        """One step's graph -> [(raw, smoothed, inter)] per object.  part: a partial step (row f17), whose compact batch of
        part.b sequences runs the same bodies on gathered state rows (_compact_fn) under the names part.name(...).
        check: a refine step replays its verifying variant (row f20)."""
        est, K = self.est, self.K
        st = self._tables()
        self._to(True)
        S, pending, f32 = (self.S, self._pending, self._f32) if part is None else (part.b, part.pending, part.f32)
        rows = (lambda n: n) if part is None else part.name
        drawer = self._drawer if part is None or self._drawer is None else self._drawer.for_sequences(part.b)
        full = kind == 'full'
        plan, reinit, b, pick = fr.FramePlan(fr.size_pattern(imgs)), None, 0, None
        draw, dt, drawn, named = draw_inputs(drawer, est.detector, plan, out, None if part is None else part.a)
        dev = est.detector.device
        if self._prev is None and (part is not None or kind == 'mixed'):
            self._prev = torch.zeros(K * self.S, 12, dtype=torch.float64, device=dev)
        wrap, extra = (lambda fn: fn), []
        if part is not None:
            wrap = lambda fn: _compact_fn(fn, full)
        with torch.no_grad():
            if full:
                name, fn, fin = fr.stage(est.detector, named(rows('track_full')), wrap(self._full_fn(st=st, draw=draw)), imgs, plan)
            elif kind == 'refine':
                prev_f32 = bool(f32[0])
                base, body = f'track_refine{int(prev_f32)}', self._refine_fn(st=st, first_f32=prev_f32, draw=draw)
                if check:
                    key = self._verify.key
                    base, body = V.graph_name(base, key), V.verifying(body, self._verify_fn(st, key))
                name, fn, fin = fr.stage(est.detector, named(rows(base)), wrap(body), imgs, plan)
            else:
                reinit, b, extra = _mixed_inputs(S, K, pending, f32, est.cfg['refine_iter'], self.refine_iter, dev, plan)
                if plan.mixed:                   # one graph per size pattern and per-size buckets (row f13)
                    _, blocks, pick = _size_buckets(reinit, plan)
                    name, fn = named(rows((plan.key('track_mixed'), tuple(blocks)))), self._mixed_fn(st, b, blocks, draw, S)
                else:
                    name, fn = named(rows(f'track_mixed{b}')), self._mixed_fn(st, b, draw=draw, S=S)
                name, fn, fin = fr.bind(est.detector, name, wrap(fn), imgs, plan)
            if part is not None:
                state = [self._prev, self._ring, self._count] + part.graph_inputs(dev)
            else:
                state = [self._ring, self._count] if full else [self._prev, self._ring, self._count]
            cams = est.detector._to_dev(glue.cameras(Ks))
            buf, poses_dev, ring, count = self.stages.run(name, fn, fin + [cams] + state + extra + dt)
            self._prev = poses_dev.clone()
            self._ring.copy_(ring)
            self._count.copy_(count)
            host = est.detector._to_host(buf)                        # the step's one synchronising read
        prev_f32 = bool(f32[0])
        if part is None:
            self._f32[:] = True
        else:
            self._f32[part.seq] = True
        if check:
            host, checked = V.split(host, K * S)
        res = self._unpack(host, kind, S, prev_f32, reinit, b, pick)
        for o, (_, _, inter) in enumerate(res):
            if drawn is not None:
                inter['drawn'] = drawn
            if check:
                inter['verify'] = {k: v[o * S:(o + 1) * S] for k, v in checked.items()}
        return res

    def _unpack(self, host, kind, S, prev_f32=False, reinit=None, b=0, pick=None):
        """A step's read -> [(raw poses float32 [S,3,4], smoothed poses float64 [S,3,4], inter)] per object.  S: the step's
        sequences (a partial step's compact batch); prev_f32: a refine step's previous poses hold float32 values.  A mixed
        step's reinit (the re-initialised sequences), b (its bucket, the gathered rows per object) and pick (the gathered
        row of each re-initialised sequence, per-size buckets; None: the first len(reinit) rows)."""
        est, K, num, n = self.est, self.K, self.num, self.K * S
        full, mixed = kind == 'full', kind == 'mixed'
        F, r = est.cfg['refine_iter'], self.refine_iter
        n_chain = 1 + (max(F, r) if mixed else F if full else r)
        qn = b if mixed else S if full else 0                   # detected rows per object
        pick = slice(0, len(reinit) if mixed else qn) if pick is None else pick
        res = est.cfg['ref_resolution']
        crop_bytes = K * qn * res * res * 3
        f64 = host[:len(host) - crop_bytes].view(np.float64)
        crops = host[len(host) - crop_bytes:].reshape(K, qn, res, res, 3)
        off = 0

        def take(m):
            nonlocal off
            off += m
            return f64[off - m:off]
        chain = take(n_chain * n * 12).reshape(n_chain, K, S, 3, 4)
        smoothed = take(n * 12).reshape(K, S, 3, 4)
        avg = take(n * 16).reshape(K, S, 8, 2)
        ring_h = take(n * num * 16).reshape(K, S, num, 8, 2).astype(np.float32)
        count_h = take(n).reshape(K, S).astype(np.int64)
        out = []
        for o, n_sel in enumerate(self._ref_counts()):
            refined = [c.astype(np.float32) for c in chain[1:, o]]
            first = chain[0, o].astype(np.float32) if (kind == 'refine' and prev_f32) else chain[0, o].copy()
            inter = {'reinit': reinit.astype(np.int64)} if mixed else {}
            if qn:
                d = take(qn * 4).reshape(qn, 4)[pick].astype(np.float32)
                idx = take(qn)[pick].astype(np.int64)
                sel_out = take(qn * 2).reshape(qn, 2)[pick].astype(np.float32)
                logits = take(qn * n_sel).reshape(qn, -1)[pick].astype(np.float32)
                inter.update({'det_position': d[:, :2].copy(), 'det_scale_r2q': d[:, 2].copy(), 'det_score': d[:, 3].copy(),
                              'det_que_img': crops[o, pick].copy(), 'sel_angle_r2q': sel_out[:, 0].copy(), 'sel_scores': logits,
                              'sel_ref_idx': idx})
            inter['refine_poses'] = [first] + refined
            inter['bbox_pts'] = ring_h[o, np.arange(S), count_h[o] - 1].copy()
            inter['smoothed_pts'] = avg[o].copy()
            out.append(((refined[-1] if refined else first), smoothed[o].copy(), inter))
        return out

    def _decode(self, host, full, prev_f32, S=None):
        """step()'s result from the read of a full step (full true) or a refine step over S sequences (default: all)."""
        return self._results(self._unpack(host, 'full' if full else 'refine', S or self.S, prev_f32))

    def _decode_mixed(self, host, reinit, b, pick=None, S=None):
        """step()'s result from the read of a mixed step over S sequences (default: all)."""
        return self._results(self._unpack(host, 'mixed', S or self.S, False, reinit, b, pick))

    def _mixed_fn(self, st, b, blocks=None, draw=None, S=None):
        """The mixed step's graph body (_mixed_fn) for S sequences (default: the tracker's) and bucket b."""
        views, R = self._groups(st)
        return _mixed_fn(self.K, S or self.S, b, self.est.cfg['refine_iter'], self.refine_iter, self._initial(st), views, R,
                         self.est.refiner._refine_warped(128), self._smoother(), blocks, draw)

    # -------------------------------------------------------------- what differs between the estimator and an object set
    def _check(self):
        if self.est._generation() != self._gen:
            raise RuntimeError('this tracker is stale: the estimator was rebuilt (build() on another object) or its weights '
                               'changed since the tracker was created; create a new one with est.tracker()')

    def _start_poses(self, poses, sequences):
        """start()'s arguments -> (the sequences, their poses float64 [K*n,12] object-major, whether they are float32)."""
        poses = np.asarray(poses)
        if sequences is None:
            if poses.shape != (self.S, 3, 4):
                raise ValueError(f'start: expected poses [{self.S},3,4], got {poses.shape}')
            seqs = np.arange(self.S)
        else:
            seqs = _sequences(self.S, sequences)
            if poses.shape != (len(seqs), 3, 4):
                raise ValueError(f'start: expected poses [{len(seqs)},3,4] for sequences {seqs.tolist()}, got {poses.shape}')
        return seqs, np.asarray(poses, np.float64).reshape(len(seqs), 12), poses.dtype == np.float32

    def _results(self, res):
        """The per-object results -> step()'s: the one object's, with predict_batch's detection entries (no det_score)."""
        (raw, smoothed, inter), = res
        inter.pop('det_score', None)
        return raw, smoothed, inter

    def _ref_counts(self):
        """The selector references of each object: the width of its sel_scores."""
        return [len(self.est.ref_info['poses'])]

    def _tables(self):
        return self.est._glue_state()

    def _groups(self, st):
        """-> (the refiner's view table of each object, the reference views per table)."""
        return [st['views']], st['tables']['ref_num']

    def _smoother(self):
        """-> smooth(poses, poses_are_f32, Ks, ring, count) -> (smoothed, averaged corners): the smoothing launch."""
        if self._dev is None:
            dev = self.est.detector.device
            self._dev = {'bbox': torch.from_numpy(self.bbox).to(dev), 'weights': torch.from_numpy(self.weights.copy()).to(dev)}
        c = self._dev
        return lambda poses, f32, Ks, ring, count: ops.track_smooth(poses, f32, c['bbox'], Ks, ring, count, c['weights'])

    def _initial(self, st):
        """The mixed step's detection: fn(frames, cams) -> (initial poses [K*b,12], crops, [the detection and selection
        tensors, in packing order])."""
        initial = self.est._initial_poses_device_fn(st)

        def fn(frames, cams):
            poses, det, crop, idx, sel_out, logits = initial(frames, cams)
            return poses, crop, [det, idx, sel_out, logits]
        return fn

    def _verify_fn(self, st, key):
        return self.est._verify_fn(st, key)

    def _full_fn(self, st, draw=None):
        predict, smooth = self.est._predict_device_fn(st), self._smoother()

        def fn(frames, cams, ring, count, *dt):
            chain, det, crop, idx, sel_out, logits = predict(frames, cams)
            poses = chain[-1]
            Ks = cams[:, :9].contiguous()
            smoothed, avg = smooth(poses, chain.shape[0] > 1, Ks, ring, count)
            if dt:
                draw(frames, poses, chain.shape[0] > 1, smoothed, Ks, dt[0])
            packed = torch.cat([t.reshape(-1).to(torch.float64) for t in (chain, smoothed, avg, ring, count, det, idx, sel_out, logits)])
            return torch.cat([packed.view(torch.uint8), crop.reshape(-1)]), poses, ring, count
        return fn

    def _refine_fn(self, st, first_f32, draw=None):
        est, iters, smooth = self.est, self.refine_iter, self._smoother()
        R, refine = st['tables']['ref_num'], est.refiner._refine_warped(128)

        def fn(frames, cams, prev, ring, count, *dt):
            poses, chain = prev, [prev]
            for it in range(iters):
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems(st['views'], R, cams, frames, poses,
                                                                                             first_f32 or it > 0)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)
                poses = ops.glue_apply_refinements(st['views'], que_pose, que_K, rect, out)
                chain.append(poses)
            Ks = cams[:, :9].contiguous()
            smoothed, avg = smooth(poses, True, Ks, ring, count)
            if dt:
                draw(frames, poses, True, smoothed, Ks, dt[0])
            packed = torch.cat([t.reshape(-1).to(torch.float64) for t in (torch.stack(chain, 0), smoothed, avg, ring, count)])
            return packed.view(torch.uint8), poses, ring, count
        return fn


# ------------------------------------------------------------------------------------------ several objects
class ObjectTracker(Tracker):
    """Every object of an ObjectSet tracked through S sequences in lockstep; see ObjectSet.tracker().

    Per object the semantics are Tracker's: the first step (and the first after reset()) is the set's full prediction
    with cfg['refine_iter'] refinements, every later step `refine_iter` refinements from the previous poses, each followed
    by predict.py's smoothing.  Rows are object-major (row o*S + s is object o on sequence s), and each step is ONE
    captured graph: refine_iter x (g6d_glue_refine_problems_objects -> one refiner stage over all K*S poses ->
    g6d_glue_apply_refinements_objects), then g6d_track_smooth_objects, so the number of launches does not grow with
    K.  The previous poses [K*S,12], the corner histories and their counts stay on the device between steps.

    start(poses, sequences) takes {name: [S,3,4]} (every object of the set, one dtype for all; [len(sequences),3,4] each
    with sequences).  step() takes Tracker.step's arguments, Ks [S,3,3] shared by all objects and out= drawing every
    object's box on its sequence's frame in object order, and returns {name: (raw poses float32 [S,3,4], smoothed poses
    float64 [S,3,4], inter)}: inter has Tracker.step's keys, and a full-prediction step adds those of ObjectSet.predict
    (det_score included); a mixed step adds 'reinit' and those entries for the re-initialised sequences.  sequences=
    steps every object on each listed sequence.  With verify_every, a verifying refine step adds inter['verify'] to every
    object's results (its windows detected against that object's references only), and a sequence is re-initialised if
    any of its objects is judged lost."""
    _host = False                    # an object set runs on the device pipeline only

    def __init__(self, objs, num_sequences, refine_iter=1, smooth_num=5, smooth_std=2.5, bboxes=None, draw=None,
                 draw_colors=None, verify_every=None, lost_score=None, lost_gate=None):
        kinds = dr.parse_kinds(draw)
        self._setup(objs.est, num_sequences, refine_iter, smooth_num, smooth_std, verify_every, lost_score, lost_gate)
        objs._check()
        boxes = object_bboxes(objs, bboxes)
        self.objs, self.names = objs, objs.names
        self.K = len(self.names)
        self.bboxes = np.ascontiguousarray(np.stack(boxes, 0))
        self._membership = objs.membership
        dev = self.est.detector.device
        self._dev = {'bboxes': torch.from_numpy(self.bboxes).to(dev), 'weights': torch.from_numpy(self.weights.copy()).to(dev)}
        self.draw = kinds
        self._drawer = dr.StepDrawer(kinds, dr.object_colors(self.names, draw_colors), self.bboxes, range(self.K), self.S,
                                     dev) if kinds else None
        self.reset()

    def _check(self):
        if self.objs.membership != self._membership:
            raise RuntimeError('this tracker is stale: objects were added to or removed from the set since it was created; '
                               'create a new one with objs.tracker()')
        self.objs._check()

    def _start_poses(self, poses, sequences):
        missing = [n for n in self.names if n not in poses]
        extra = sorted(set(poses) - set(self.names))
        if missing or extra:
            raise ValueError(f'start: need poses for exactly the set\'s objects {self.names}; missing {missing}, unknown {extra}')
        seqs = np.arange(self.S) if sequences is None else _sequences(self.S, sequences)
        arrs = [np.asarray(poses[n]) for n in self.names]
        for n, a in zip(self.names, arrs):
            if a.shape != (len(seqs), 3, 4):
                raise ValueError(f'start: object {n!r}: expected poses [{len(seqs)},3,4], got {a.shape}')
        dtypes = {a.dtype for a in arrs}
        if len(dtypes) != 1:
            raise ValueError(f'start: the objects\' poses have different dtypes {sorted(str(d) for d in dtypes)}; the refinement '
                             'reads them all as float32 or all as float64, so pass one dtype')
        return seqs, np.concatenate(arrs, 0).astype(np.float64).reshape(-1, 12), arrs[0].dtype == np.float32

    def _results(self, res):
        return dict(zip(self.names, res))

    def _ref_counts(self):
        return [len(ob.ref_info['poses']) for ob in self.objs._objects.values()]

    def _tables(self):
        return None

    def _groups(self, st):
        objs = list(self.objs._objects.values())
        return [ob.tables['views'] for ob in objs], objs[0].tables['tables']['ref_num']

    def _smoother(self):
        c = self._dev
        return lambda poses, f32, Ks, ring, count: ops.track_smooth_objects(poses, f32, c['bboxes'], Ks, ring, count,
                                                                            c['weights'])

    def _detections(self, det, sels):
        """The set's detections [K*n,4] and selections [(idx, sel_out, logits)] per object -> the tensors a step packs
        after its state, object by object."""
        n, parts = det.shape[0] // self.K, []
        for o in range(self.K):
            parts += [det[o * n:(o + 1) * n], *sels[o]]
        return parts

    def _initial(self, st):
        initial = self.objs._initial_poses_device_fn()

        def fn(frames, cams):
            poses, det, sels, crop = initial(frames, cams)          # the set's shared detection on the gathered frames
            return poses, crop, self._detections(det, sels)
        return fn

    def _verify_fn(self, st, key):
        return self.objs._verify_fn(key)

    # the graph bodies take the estimator's tables as st= (Tracker's driver passes them by keyword): the set's objects
    # hold their own, so st is None here
    def _full_fn(self, draw=None, st=None):
        predict, smooth = self.objs._predict_device_fn(), self._smoother()

        def fn(frames, cams, ring, count, *dt):
            chain, det, sels, crop = predict(frames, cams)
            poses = chain[-1]
            Ks = cams[:, :9].contiguous()
            smoothed, avg = smooth(poses, chain.shape[0] > 1, Ks, ring, count)
            if dt:
                draw(frames, poses, chain.shape[0] > 1, smoothed, Ks, dt[0])
            parts = [chain, smoothed, avg, ring, count] + self._detections(det, sels)
            packed = torch.cat([t.reshape(-1).to(torch.float64) for t in parts])
            return torch.cat([packed.view(torch.uint8), crop.reshape(-1)]), poses, ring, count
        return fn

    def _refine_fn(self, first_f32, draw=None, st=None):
        (views, R), iters, smooth = self._groups(st), self.refine_iter, self._smoother()
        refine = self.est.refiner._refine_warped(128)

        def fn(frames, cams, prev, ring, count, *dt):
            poses, chain = prev, [prev]
            for it in range(iters):
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_objects(views, R, cams, frames, poses,
                                                                                                     first_f32 or it > 0)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)           # one refiner stage for all K*S poses
                poses = ops.glue_apply_refinements_objects(views, que_pose, que_K, rect, out)
                chain.append(poses)
            Ks = cams[:, :9].contiguous()
            smoothed, avg = smooth(poses, True, Ks, ring, count)
            if dt:
                draw(frames, poses, True, smoothed, Ks, dt[0])
            packed = torch.cat([t.reshape(-1).to(torch.float64) for t in (torch.stack(chain, 0), smoothed, avg, ring, count)])
            return packed.view(torch.uint8), poses, ring, count
        return fn
