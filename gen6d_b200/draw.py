"""Drawn frames on the device (DESIGN.md row f16): predict.py's images_out / images_out_smooth, i.e. each frame with the
object's 3-D box drawn by utils/draw_utils.py draw_bbox_3d, bit for bit with OpenCV, into RGB tensors or NV12 surfaces.

- draw_boxes(frames, Ks, poses, bbox_3d): an eager call on CUDA RGB frames, e.g. for predict_batch's results;
- Gen6DEstimator.tracker(..., draw='raw' / 'smoothed' / ('raw', 'smoothed')): every step draws inside its captured
  graph, as the graph's last node (g6d_draw_boxes), from the working frame the graph already holds.

The raw box is projected with the raw float32 pose in float32 (the corners inter['bbox_pts'] holds), the smoothed box
with the float64 smoothed pose in float64 (predict.py's pts__), then rounded as np.round(...).astype(np.int32).
"""
import copy
import ctypes as C

import numpy as np
import torch

from . import _lib, ops
from .frames import NV12

KINDS = ('raw', 'smoothed')
DEFAULT_COLOR = (0, 0, 255)


def parse_kinds(draw):
    """draw -> the kinds to draw in KINDS order (a tuple), or None; ValueError for anything else."""
    if draw is None:
        return None
    kinds = (draw,) if isinstance(draw, str) else tuple(draw)
    bad = [k for k in kinds if k not in KINDS]
    if bad or not kinds or len(set(kinds)) != len(kinds):
        raise ValueError(f"draw must be 'raw', 'smoothed' or ('raw', 'smoothed'), got {draw!r}")
    return tuple(k for k in KINDS if k in kinds)


def parse_color(color, what='draw_color'):
    c = tuple(int(v) for v in color)
    if len(c) != 3 or not all(0 <= v <= 255 for v in c):
        raise ValueError(f'{what} must be an (R, G, B) triple of 0..255, got {color!r}')
    return c


def object_colors(names, draw_colors):
    """draw_colors {name: (R, G, B)} -> the edge colour of every object in set order (DEFAULT_COLOR where not given)."""
    draw_colors = dict(draw_colors or {})
    unknown = sorted(set(draw_colors) - set(names))
    if unknown:
        raise ValueError(f'draw_colors names objects that are not in the set: {unknown} (objects: {list(names)})')
    return [parse_color(draw_colors.get(n, DEFAULT_COLOR), f'draw_colors[{n!r}]') for n in names]


def dst_row(d, h, w, device, what):
    """A destination (CUDA uint8 RGB tensor [h, w, 3] with any row pitch, or an NV12 of even size h x w) -> DeviceFrame."""
    def plane(t, name, shape, unit):
        if not isinstance(t, torch.Tensor) or t.device != device or t.dtype != torch.uint8 or list(t.shape) != shape:
            got = f'{t.dtype} {list(t.shape)} on {t.device}' if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f'{what}: {name} must be a uint8 {shape} tensor on {device} (the working size), got {got}')
        if (len(shape) == 3 and t.stride(2) != 1) or (shape[1] > 1 and t.stride(1) != unit) or (shape[0] > 1 and t.stride(0) < unit * shape[1]):
            raise ValueError(f'{what}: {name} has strides {list(t.stride())}; need unit column steps and a row pitch >= {unit} x width')
    if isinstance(d, NV12):
        if h % 2 or w % 2:
            raise ValueError(f'{what}: an NV12 destination needs an even working size, the frame is {h} x {w}')
        plane(d.y, 'the NV12 Y plane', [h, w], 1)
        plane(d.uv, 'the NV12 UV plane', [h // 2, w], 1)
        return ops.DeviceFrame(d.y.data_ptr(), d.uv.data_ptr(), d.y.stride(0) if h > 1 else w, d.uv.stride(0) if h > 2 else w,
                               h, w, _lib.G6D_FRAME_NV12, 0)
    plane(d, 'an RGB destination', [h, w, 3], 3)
    return ops.DeviceFrame(d.data_ptr(), None, d.stride(0) if h > 1 else 3 * w, 0, h, w, _lib.G6D_FRAME_RGB, 0)


def _bytes(rows, cls):
    return np.frombuffer(bytes((cls * len(rows))(*rows)), np.uint8)


def _upload(a, device):
    return torch.from_numpy(np.array(a, copy=True, order="C")).to(device)


class StepDrawer:
    """The draw node of a tracker's step graphs.  The tracker's rows are group-major, row g*S + s being group g (an object,
    an instance slot, or slot m of object o as group m*K + o) on sequence s; group g draws box bbox_of[g] in
    colors[bbox_of[g]], every group of a sequence on that sequence's frame in row order.  live: the groups are instance
    slots, drawn only while their track id (a graph tensor) is >= 0.  Destinations are kind-major (destination k*S + s
    shows sequence s), named by a graph input of DeviceFrame rows, so new allocations replay the same graph."""

    def __init__(self, kinds, colors, bboxes, bbox_of, S, device, live=False):
        self.kinds, self.S, self.device, self.live = kinds, S, torch.device(device), live
        self.G, self.bbox_of, self.colors = len(bbox_of), list(bbox_of), [parse_color(c) for c in colors]
        if self.G > _lib.G6D_DRAW_MAX_BOXES:
            raise ValueError(f'draw: {self.G} boxes per frame (objects x instance slots); at most {_lib.G6D_DRAW_MAX_BOXES} are drawn')
        self.bboxes = torch.from_numpy(np.ascontiguousarray(bboxes, np.float32).reshape(-1, 8, 3)).to(device)
        self._srcs, self._boxes, self._own, self._subs = {}, {}, {}, {}

    def name(self, base):
        """The graph name of a drawing step: apart from the non-drawing graph `base`."""
        return (base, 'draw', self.kinds)

    def src_table(self, module, plan):
        """The sources of the frames tensor a graph body sees: [qn, h, w, 3] (one size) or the canvas [qn, H, W, 3]."""
        t = self._srcs.get(plan.pattern)
        if t is None:
            H, W = (plan.H, plan.W) if plan.mixed else plan.pattern[0]
            rows = [ops.DrawSrc(i * H * W * 3, W * 3, h, w) for i, (h, w) in enumerate(plan.pattern)]
            t = self._srcs[plan.pattern] = (module._to_dev(_bytes(rows, ops.DrawSrc)), rows)
        return t

    def box_table(self, module, raw_f32):
        t = self._boxes.get(raw_f32)
        if t is None:
            S, G, rows = self.S, self.G, []
            for k, kind in enumerate(self.kinds):
                f32 = int(raw_f32) if kind == 'raw' else 0
                for s in range(S):
                    for g in range(G):           # poses: [raw [G*S,12]; smoothed [G*S,12]], row g*S + s
                        b = self.bbox_of[g]
                        rows.append(ops.DrawBox(k * S + s, KINDS.index(kind) * G * S + g * S + s, s, b, f32,
                                                g * S + s if self.live else -1, (C.c_uint8 * 4)(*self.colors[b], 0)))
            t = self._boxes[raw_f32] = (module._to_dev(_bytes(rows, ops.DrawBox)), rows)
        return t

    def for_sequences(self, S):
        """The drawer of a compact batch of S sequences (a partial step, row f17): this drawer's kinds, boxes and colours,
        its own tables and buffers; made once per S."""
        sub = self._subs.get(S)
        if sub is None:
            sub = self._subs[S] = copy.copy(self)
            sub.S, sub._srcs, sub._boxes, sub._own, sub._subs = S, {}, {}, {}, {}
        return sub

    def destinations(self, module, plan, out, real=None):
        """-> (the DeviceFrame table on the device, inter['drawn'] or None), checked before anything is enqueued.  out
        None: tracker-owned RGB buffers per size pattern (their table is made once).  real: out holds destinations for
        the first `real` sequences only (a partial step's listed ones); the others (its padding) draw into the
        tracker-owned buffers as scratch."""
        S, pattern = self.S, plan.pattern
        real = S if real is None else real
        if out is None or real < S:
            own = self._own.get(pattern)
            if own is None:
                bufs = {k: [torch.empty(h, w, 3, dtype=torch.uint8, device=self.device) for h, w in pattern] for k in self.kinds}
                own = self._own[pattern] = (self._table(module, plan, bufs), bufs)
            if out is None:
                return own[0], {k: list(v) for k, v in own[1].items()}
        if not isinstance(out, dict) or set(out) != set(self.kinds):
            raise ValueError(f'step: out must be a dict with exactly the drawn kinds {list(self.kinds)}, got '
                             f'{sorted(out) if isinstance(out, dict) else type(out).__name__}')
        for k in self.kinds:
            if len(out[k]) != real:
                raise ValueError(f'step: out[{k!r}] holds {len(out[k])} destinations, need one per sequence ({real})')
        if real < S:
            out = {k: list(out[k]) + own[1][k][real:] for k in self.kinds}
        return self._table(module, plan, out), None

    def _table(self, module, plan, dests):
        rows = [dst_row(dests[k][s], h, w, self.device, f'step: out[{k!r}][{s}]') for k in self.kinds
                for s, (h, w) in enumerate(plan.pattern)]
        srcs, boxes = self.src_table(module, plan)[1], self.box_table(module, True)[1]
        self.box_table(module, False)                   # both tables exist before a graph captures them
        n = self.G * self.S
        ops.draw_check((ops.DrawSrc * self.S)(*srcs), (ops.DrawBox * len(boxes))(*boxes), (ops.DeviceFrame * len(rows))(*rows),
                       len(KINDS) * n, self.S, len(self.bboxes), n if self.live else 0)
        return module._to_dev(_bytes(rows, ops.DeviceFrame))

    def node(self, module, plan, frames, raw, raw_f32, smoothed, Ks, table, ids=None):
        """Inside the graph, after the smoothing: draw every kind of every sequence into the destinations of `table`.
        raw / smoothed: float64 [G*S,12]; Ks: the contiguous float64 [S,9] the smoothing read; ids: int64 [G*S] (live)."""
        srcs, boxes = self.src_table(module, plan)[0], self.box_table(module, raw_f32)[0]
        poses = torch.cat([raw, smoothed], 0)
        n_dst = len(self.kinds) * self.S
        max_rows, max_cols = max(h for h, _ in plan.pattern), max(w for _, w in plan.pattern)
        ops.draw_boxes(frames.data_ptr(), srcs, self.S, poses, Ks, self.bboxes, boxes, boxes.numel() // C.sizeof(ops.DrawBox), table,
                       n_dst, max_rows, max_cols, ids if self.live else None)


def draw_boxes(frames, Ks, poses, bbox_3d, color=DEFAULT_COLOR, out=None):
    """predict.py's draw_bbox_3d(frame, project_points(bbox_3d, pose, K), color) on CUDA uint8 RGB frames [h, w, 3] (any
    row pitch), every box of a frame drawn one after the other.  poses: per frame a pose [3,4] or poses [n,3,4] (e.g.
    predict_batch's rows, or an instance list); their dtype picks the projection as in predict.py: float32 poses in
    float32 (images_out), float64 in float64 (images_out_smooth).  Ks: per frame [3,3].  out: per frame a destination
    (CUDA RGB tensor or NV12 of the frame's size); None: new RGB tensors.  Returns the destinations."""
    frames, Ks = list(frames), list(Ks)
    if not frames or len(Ks) != len(frames) or len(poses) != len(frames):
        raise ValueError(f'draw_boxes: {len(frames)} frames, {len(Ks)} Ks and {len(poses)} pose sets; need one of each per frame')
    dev = frames[0].device if isinstance(frames[0], torch.Tensor) else None
    srcs, base = [], None
    for i, f in enumerate(frames):
        if not isinstance(f, torch.Tensor) or not f.is_cuda or f.device != dev:
            raise ValueError(f'draw_boxes: frame {i} must be a CUDA uint8 RGB tensor on one device')
        dst_row(f, int(f.shape[0]) if f.dim() == 3 else -1, int(f.shape[1]) if f.dim() == 3 else -1, dev, f'draw_boxes: frame {i}')
    base = min(f.data_ptr() for f in frames)
    for f in frames:
        h, w = int(f.shape[0]), int(f.shape[1])
        srcs.append(ops.DrawSrc(f.data_ptr() - base, f.stride(0) if h > 1 else 3 * w, h, w))
    color = parse_color(color, 'color')
    box = np.ascontiguousarray(bbox_3d, np.float32).reshape(1, 8, 3)
    pose_rows, K_rows, boxes = [], [], []
    for i, (p, K) in enumerate(zip(poses, Ks)):
        p = np.asarray(p)
        if p.shape[-2:] != (3, 4):
            raise ValueError(f'draw_boxes: frame {i} poses are {list(p.shape)}; need [3,4] or [n,3,4]')
        K_rows.append(np.asarray(K, np.float64).reshape(9))
        for q in p.reshape(-1, 3, 4):
            boxes.append(ops.DrawBox(i, len(pose_rows), i, 0, int(p.dtype == np.float32), -1, (C.c_uint8 * 4)(*color, 0)))
            pose_rows.append(np.asarray(q, np.float64).reshape(12))
    if out is None:
        out = [torch.empty(int(f.shape[0]), int(f.shape[1]), 3, dtype=torch.uint8, device=dev) for f in frames]
    elif len(out) != len(frames):
        raise ValueError(f'draw_boxes: out holds {len(out)} destinations for {len(frames)} frames')
    rows = [dst_row(d, s.rows, s.cols, dev, f'draw_boxes: out[{i}]') for i, (d, s) in enumerate(zip(out, srcs))]
    n = len(frames)
    st, bt, dt = (ops.DrawSrc * n)(*srcs), (ops.DrawBox * max(len(boxes), 1))(*boxes), (ops.DeviceFrame * n)(*rows)
    ops.draw_check(st, (ops.DrawBox * len(boxes))(*boxes), dt, max(len(pose_rows), 1), n, 1)
    pz = _upload(np.stack(pose_rows) if pose_rows else np.zeros((1, 12)), dev)
    ops.draw_boxes(base, _upload(_bytes(srcs, ops.DrawSrc), dev), n, pz, _upload(np.stack(K_rows), dev),
                   torch.from_numpy(box).to(dev), _upload(np.frombuffer(bytes(bt), np.uint8)[:len(boxes) * C.sizeof(ops.DrawBox)], dev),
                   len(boxes), _upload(_bytes(rows, ops.DeviceFrame), dev), n, max(s.rows for s in srcs), max(s.cols for s in srcs))
    return out
