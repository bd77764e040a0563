"""Frames of different sizes in one batch or tracker step (DESIGN.md row f13).

Frame size matters to two things on the device path only:

- the crops between the stages, cut by the warp kernels from g6d_warp_job records the glue kernels fill from
  `frames + i*rows*cols*3`.  A batch of mixed sizes hands them a zero-padded canvas [qn, H, W, 3] (g6d_frames_canvas,
  the first node of the captured graph); every crop cut from it equals the crop of the true-size frame bit for bit;
- the detector, whose pyramid, correlation and heads depend on (h, w).  Its step runs once per distinct size on that
  size's frames at their true size, a contiguous [g, h, w, 3] view of the packed input, and per_size scatters its rows
  back to frame order.  Everything after detection keeps the single-size row layout.

The frames are grouped by size (groups in order of first appearance, input order inside a group) and packed in group
order into one buffer, each group at a 256-byte-aligned offset, and uploaded with one copy.  The size pattern (the
(h, w) of every frame) goes into every graph name: the graph caches key on input shapes only, and two patterns with the
same packed length would otherwise share a graph.  A batch of one size takes none of this: the caller keeps its
single-size path and graphs.
"""
import threading
from contextlib import contextmanager

import numpy as np
import torch

from . import ops

ALIGN = 256          # byte alignment of every size group in the packed input


def check_frames(que_imgs, que_Ks, what):
    """-> the frames as numpy arrays; ValueError unless there is at least one frame, one K per frame and every frame is
    uint8 [h, w, 3]."""
    frames = [np.asarray(f) for f in que_imgs]
    if not frames or len(que_Ks) != len(frames):
        raise ValueError(f'{what}: {len(frames)} frames and {len(que_Ks)} intrinsics; need one K per frame and at least one frame')
    for i, f in enumerate(frames):
        if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 or f.shape[0] < 1 or f.shape[1] < 1:
            raise ValueError(f'{what}: frame {i} is {f.dtype} {list(f.shape)}; frames must be uint8 [h, w, 3]')
    return frames


def size_pattern(frames):
    """The (h, w) of every frame, in input order."""
    return tuple((int(f.shape[0]), int(f.shape[1])) for f in frames)


def is_mixed(frames):
    return len(set(size_pattern(frames))) > 1


def require_one_size(frames, what):
    """ValueError for frames of different sizes on a path that takes one size (raised before anything is uploaded)."""
    if is_mixed(frames):
        raise ValueError(f'{what} needs frames of one size, got sizes {sorted(set(size_pattern(frames)))}: frames of different '
                         "sizes go through the device pipeline only (cfg['device_glue'] on, cfg['host_warps'] off)")


class FramePlan:
    """How a batch of frames of different sizes is packed: groups [(h, w, frame indices, byte offset)] in order of first
    appearance, `table` [(byte offset, rows, cols)] per frame, the canvas size (H, W), the packed length `nbytes` and
    `order`, the frame indices in group order (the device index every scatter reads)."""

    def __init__(self, pattern):
        self.pattern = tuple((int(h), int(w)) for h, w in pattern)
        if not self.pattern:
            raise ValueError('a frame plan needs at least one frame')
        self.groups, table, off = [], [None] * len(self.pattern), 0
        for h, w in dict.fromkeys(self.pattern):
            idx = np.asarray([i for i, s in enumerate(self.pattern) if s == (h, w)], np.int64)
            self.groups.append((h, w, idx, off))
            for j, i in enumerate(idx):
                table[i] = (off + j * h * w * 3, h, w)
            off += -(-len(idx) * h * w * 3 // ALIGN) * ALIGN
        self.table, self.nbytes = table, off
        self.H, self.W = max(h for h, _ in self.pattern), max(w for _, w in self.pattern)
        self.order = np.concatenate([g[2] for g in self.groups])
        self.mixed = len(self.groups) > 1

    def key(self, name):
        """The graph name of `name` for this size pattern."""
        return (name, 'sizes', self.pattern)

    def upload(self, module, frames):
        """-> graph inputs [packed u8 [nbytes], order int64 [qn]] on the device: one pinned staging copy each."""
        arrays = [frames[i] for _, _, idx, _ in self.groups for i in idx]
        offsets = [self.table[i][0] for _, _, idx, _ in self.groups for i in idx]
        return [module.upload_packed(arrays, offsets, self.nbytes), module._to_dev(self.order)]


def stage(module, name, fn, frames, plan=None):
    """A graph body fn(frames u8 [qn,h,w,3], *rest) and the numpy frames -> (graph name, graph body, frame inputs) for
    StageCache.run(name, fn, frame inputs + rest).  One size: (name, fn, [the frames uploaded as [qn,h,w,3]]), exactly
    the single-size path; several: the pattern's name, on_canvas(fn) and the packed upload."""
    plan = plan or FramePlan(size_pattern(frames))
    if not plan.mixed:
        return name, fn, [module.upload_frame(frames)]
    return plan.key(name), on_canvas(fn, plan), plan.upload(module, frames)


# ------------------------------------------------------------------------------------------ detection per size
_tls = threading.local()


def _registry():
    reg = getattr(_tls, 'reg', None)
    if reg is None:
        reg = _tls.reg = {}
    return reg


@contextmanager
def _registered(frames, groups):
    """While active, per_size(detect, frames) runs detect once per group: groups [(u8 [g,h,w,3], dst rows int64 [g])]."""
    reg = _registry()
    reg[id(frames)] = (frames, groups)
    try:
        yield
    finally:
        reg.pop(id(frames), None)


def scatter_rows(parts, dsts, n):
    """Per group a tensor of L*g rows (slot l of the group's frame j at row l*g + j) -> one tensor of L*n rows with that
    row at l*n + dsts[group][j]: the (slot, frame) rows of the frame-major (L = 1), object-major (L = K) and
    instance-major (L = M or M*K) layouts, back in frame order."""
    L = parts[0].shape[0] // dsts[0].numel()
    out = parts[0].new_empty((L * n,) + tuple(parts[0].shape[1:]))
    for p, dst in zip(parts, dsts):
        rows = (torch.arange(L, device=dst.device, dtype=torch.int64)[:, None] * n + dst[None, :]).reshape(-1)
        out.index_copy_(0, rows, p)
    return out


def per_size(detect, frames):
    """detect(u8 [g,h,w,3]) -> a tensor (or tuple of tensors) of (slot, frame) rows, frame minor.  On the canvas of a mixed
    batch (or a gather of it) detect runs once per size group at the true size and the rows are scattered back to frame
    order; on any other tensor this is detect(frames)."""
    ent = _registry().get(id(frames))
    if ent is None or ent[0] is not frames:
        return detect(frames)
    groups = ent[1]
    outs = [detect(u8) for u8, _ in groups]
    single = isinstance(outs[0], torch.Tensor)
    outs = [(o,) if single else tuple(o) for o in outs]
    dsts = [dst for _, dst in groups]
    res = tuple(scatter_rows([o[k] for o in outs], dsts, frames.shape[0]) for k in range(len(outs[0])))
    return res[0] if single else res


def on_canvas(fn, plan):
    """A graph body fn(frames u8 [qn,h,w,3], *rest) -> g(packed, order, *rest) for a mixed batch: the canvas of the packed
    frames (g6d_frames_canvas) goes to fn as `frames`, with detection per size (per_size) on it."""
    def g(packed, order, *rest):
        canvas = ops.frames_canvas(packed, plan.table, plan.H, plan.W)
        groups, s = [], 0
        for h, w, idx, off in plan.groups:
            n = len(idx)
            groups.append((packed[off:off + n * h * w * 3].view(n, h, w, 3), order[s:s + n]))
            s += n
        with _registered(canvas, groups):
            return fn(canvas, *rest)
    return g


@contextmanager
def gathered(frames, sub, seq, blocks):
    """sub = frames.index_select(0, seq) with seq ordered by size group, blocks[z] rows of group z: while active, per_size
    on `sub` detects each block on the gathered true-size frames of its group.  No effect unless `frames` is the canvas
    of a mixed batch."""
    ent = _registry().get(id(frames))
    if ent is None or ent[0] is not frames:
        yield
        return
    groups = ent[1]
    inv = torch.empty(frames.shape[0], dtype=torch.int64, device=frames.device)      # frame -> its position in its group
    for u8, dst in groups:
        inv.index_copy_(0, dst, torch.arange(u8.shape[0], dtype=torch.int64, device=frames.device))
    sub_groups, s = [], 0
    for (u8, _), b in zip(groups, blocks):
        if b:
            local = inv.index_select(0, seq[s:s + b])
            sub_groups.append((u8.index_select(0, local), torch.arange(s, s + b, dtype=torch.int64, device=frames.device)))
        s += b
    with _registered(sub, sub_groups):
        yield
