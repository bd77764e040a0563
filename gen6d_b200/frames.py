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

Frames already on the GPU (row f14): a call's frames may instead all be device frames, CUDA uint8 RGB tensors [h, w, 3]
with pitched rows or NV12 decoder surfaces (NV12), in any mix of sizes.  Their bytes never cross PCIe: the graph input
is a device table of g6d_device_frame rows (plane pointers, pitches, size, format, offset in the packed layout), and
the graph's first node, g6d_frames_gather, writes the packed layout of FramePlan from them (converting NV12 as
cv2.cvtColor(COLOR_YUV2RGB_NV12) does).  From the packed buffer on, the graph is the numpy path's: the [qn, h, w, 3]
view for one size, on_canvas for several.  Pointers and pitches live in the table, so a device-frame graph keys on the
size pattern only, one size included ('device' in the name keeps it apart from the numpy graphs of that pattern), and a
new allocation or pitch replays the same graph.

Device frames at a working resolution (row f15): a device frame wrapped in Resized is resized (and rotated) to its
working size as predict.py's video2image does on the host, bit for bit with cv2.resize + cv2.rotate, by the graph's
first node, g6d_frames_gather_resized.  A call holding one takes that gather for all its frames (plain ones as identity
rows of its g6d_resized_frame table) under a 'device-resized' key on the working size pattern; the sources live in the
table, so a new decoder resolution with the same working sizes replays the same graph.
"""
import ctypes as C
import threading
from contextlib import contextmanager

import numpy as np
import torch

from . import _lib, ops

ALIGN = 256          # byte alignment of every size group in the packed input

_DEVICE_PIPELINE = "device frames (CUDA tensors, NV12) go through the device pipeline only (cfg['device_glue'] on, cfg['host_warps'] off)"


class NV12:
    """An NV12 frame on the device, as GPU decoders hand it over: y the uint8 CUDA luma plane [h, w], uv the interleaved
    (U, V) chroma plane [h/2, w], each with unit column stride and any row pitch >= w; h and w even.  It is converted as
    cv2.cvtColor(np.vstack([y, uv]), cv2.COLOR_YUV2RGB_NV12) converts it (BT.601 limited range), bit for bit.  A decoder
    surface t of [h*3/2, pitch] bytes is NV12(t[:h, :w], t[h:, :w])."""
    __slots__ = ('y', 'uv')

    def __init__(self, y, uv):
        self.y, self.uv = y, uv

    @property
    def shape(self):
        """(h, w, 3): the shape of the RGB frame it converts to."""
        return (int(self.y.shape[0]), int(self.y.shape[1]), 3)

    def __repr__(self):
        return f'NV12({self.shape[0]}x{self.shape[1]}, {self.y.device})'


_ROTATIONS = (0, 90, 180, 270)


class Resized:
    """A device frame (a CUDA uint8 RGB tensor [h, w, 3] with any row pitch, or an NV12 frame) resized and rotated to its
    working size inside the graph's first node (row f15), bit for bit as
        cv2.rotate(cv2.resize(rgb, (w', h'), interpolation=cv2.INTER_LINEAR), code)
    with rgb the frame's RGB bytes (an NV12 frame's cv2.cvtColor(COLOR_YUV2RGB_NV12) conversion).  Downscales and the
    identity only: ValueError for a working size larger than the frame on either axis.

    max_side: prepare.video2image's rule, ratio = max_side / max(h, w) and (h', w') = (int(ratio*h), int(ratio*w)) in
    Python floats; or size=(h', w'), the resized size before the rotation.  Exactly one of them.
    rotate: 0, 90, 180 or 270 degrees clockwise after the resize (cv2.ROTATE_90_CLOCKWISE, ROTATE_180,
    ROTATE_90_COUNTERCLOCKWISE).  predict.py's --transpose is rotate=180 with OpenCV >= 4.5 (flip(0) then flip(1)) and
    rotate=90 before (transpose then flip(1)).

    .shape is the working (rows, cols, 3) after the rotation: every call sees the frame at that size, and a new source
    resolution, pitch or allocation with the same working sizes replays the same graph."""
    __slots__ = ('frame', 'size', 'rotate')

    def __init__(self, frame, max_side=None, size=None, rotate=0):
        if not isinstance(frame, (torch.Tensor, NV12)):
            raise ValueError(f'Resized: frame is {type(frame).__name__}; need a CUDA uint8 RGB tensor [h, w, 3] or an NV12 frame '
                             '(numpy frames are resized on the host, as predict.py does)')
        shape = tuple(frame.shape) if isinstance(frame, torch.Tensor) else tuple(getattr(frame.y, 'shape', ())) + (3,)
        if len(shape) != 3 or shape[2] != 3 or shape[0] < 1 or shape[1] < 1:
            raise ValueError(f'Resized: frame is {list(shape)}; need [h, w, 3]')
        h, w = int(shape[0]), int(shape[1])
        if (max_side is None) == (size is None):
            raise ValueError('Resized: give exactly one of max_side and size')
        if max_side is not None:
            if not max_side > 0:
                raise ValueError(f'Resized: max_side = {max_side}, need > 0')
            ratio = max_side / max(h, w)
            size = (int(ratio * h), int(ratio * w))
        size = tuple(int(s) for s in size)
        if len(size) != 2 or min(size) < 1:
            raise ValueError(f'Resized: working size {size} of a {h} x {w} frame; need (rows, cols) >= (1, 1)')
        if size[0] > h or size[1] > w:
            raise ValueError(f'Resized: {h} x {w} -> {size[0]} x {size[1]} upscales; only downscales and the identity are '
                             'resized on the device')
        if rotate not in _ROTATIONS:
            raise ValueError(f'Resized: rotate = {rotate}; need one of {_ROTATIONS} degrees clockwise')
        self.frame, self.size, self.rotate = frame, size, int(rotate)

    @property
    def shape(self):
        """(rows, cols, 3): the working size, after the rotation."""
        h, w = self.size
        return (w, h, 3) if self.rotate in (90, 270) else (h, w, 3)

    def intrinsics(self, K):
        """A camera matrix K [3, 3] of the source frame -> the matrix that projects the same camera points into the working
        frame: OpenCV's pixel-centre convention x' = (x + 0.5) * w'/w - 0.5 (rows alike), then the rotation.  With a
        rotation the result M is not upper triangular: M = K_w @ Rz, with Rz the turn about the optical axis (the 2x2
        linear part of the pixel rotation, e.g. -I for 180) and K_w upper triangular (for a K without skew).  The
        estimator takes K_w (M @ Rz.T); its poses are then those of the camera turned by Rz.  predict.py's pseudo-K is
        built from the working size and needs no mapping."""
        h, w = int(self.frame.shape[0]), int(self.frame.shape[1])
        (rh, rw), sx, sy = self.size, self.size[1] / w, self.size[0] / h
        A = np.array([[sx, 0, 0.5 * sx - 0.5], [0, sy, 0.5 * sy - 0.5], [0, 0, 1]])
        R = {0: np.eye(3),
             90: np.array([[0, -1, rh - 1], [1, 0, 0], [0, 0, 1]], np.float64),
             180: np.array([[-1, 0, rw - 1], [0, -1, rh - 1], [0, 0, 1]], np.float64),
             270: np.array([[0, 1, 0], [-1, 0, rw - 1], [0, 0, 1]], np.float64)}[self.rotate]
        return R @ A @ np.asarray(K, np.float64)

    def __repr__(self):
        return f'Resized({self.frame!r} -> {self.size[0]}x{self.size[1]}, rotate={self.rotate})'


def _gpu_frame(f):
    return isinstance(f, (NV12, Resized)) or (isinstance(f, torch.Tensor) and f.is_cuda)


def is_device(frames):
    """True when the frames are device frames: a tensor, or a sequence holding a tensor, an NV12 or a Resized frame."""
    return isinstance(frames, torch.Tensor) or any(isinstance(f, (torch.Tensor, NV12, Resized)) for f in frames)


def has_resized(frames):
    """True when a sequence of device frames holds a Resized frame (the call takes the resized gather, row f15)."""
    return not isinstance(frames, torch.Tensor) and any(isinstance(f, Resized) for f in frames)


def host_only(que_imgs, what):
    """TypeError if any frame is on the GPU, on a path that takes numpy frames only (raised before anything is launched)."""
    if isinstance(que_imgs, torch.Tensor) and que_imgs.is_cuda or any(_gpu_frame(f) for f in que_imgs):
        raise TypeError(f'{what} takes numpy uint8 [h, w, 3] frames only: {_DEVICE_PIPELINE}')


def as_frames(que_imgs, what, module, host_path=None):
    """The frames of a call as a list: numpy arrays (np.asarray of each, the host upload path) or, when they are device
    frames, RGB tensors [h, w, 3] and NV12 frames checked to be on module.device, the network's device, which is read
    for device frames only (a [qn, h, w, 3] tensor counts as qn frames).
    ValueError for a mix of numpy and device frames or a malformed device frame, before anything is enqueued.
    host_path: None on the device pipeline, else the name of the numpy-only path the call takes (TypeError for frames
    on the GPU)."""
    if host_path is not None:
        host_only(que_imgs, host_path)
    elif is_device(que_imgs):
        frames = list(que_imgs.unbind(0)) if isinstance(que_imgs, torch.Tensor) and que_imgs.dim() == 4 else list(que_imgs)
        if isinstance(que_imgs, torch.Tensor) and que_imgs.dim() != 4:
            raise ValueError(f'{what}: a frames tensor must be [qn, h, w, 3], got {list(que_imgs.shape)}')
        for i, f in enumerate(frames):
            _check_device_frame(f, i, what, torch.device(module.device))
        return frames
    return [np.asarray(f) for f in que_imgs]


def _check_device_frame(f, i, what, device):
    def plane(t, name, rows, cols, ch):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f'{what}: frame {i}: {name} is {type(t).__name__}, not a torch tensor; a call\'s frames are all numpy '
                             'arrays or all device frames (CUDA tensors, NV12)')
        if t.device != device:
            raise ValueError(f'{what}: frame {i}: {name} is on {t.device}; device frames must be on {device}, the estimator\'s '
                             'device (numpy arrays take the host upload path)')
        if t.dtype != torch.uint8:
            raise ValueError(f'{what}: frame {i}: {name} is {t.dtype}; device frames are uint8')
        shape = [rows, cols] + ([ch] if ch else [])
        if list(t.shape) != shape or rows < 1 or cols < 1:
            raise ValueError(f'{what}: frame {i}: {name} is {list(t.shape)}, need {shape}')
        unit = 3 if ch else 1
        if (ch and t.stride(2) != 1) or (cols > 1 and t.stride(1) != unit) or (rows > 1 and t.stride(0) < unit * cols):
            raise ValueError(f'{what}: frame {i}: {name} has strides {list(t.stride())}; need unit column steps '
                             f'({"stride(2) == 1, stride(1) == 3" if ch else "stride(1) == 1"}) and a row pitch >= '
                             f'{unit} x width')

    if isinstance(f, Resized):                   # its size and rotation were checked when it was built
        _check_device_frame(f.frame, i, what, device)
    elif isinstance(f, NV12):
        h, w = int(f.y.shape[0]) if f.y.dim() == 2 else -1, int(f.y.shape[1]) if f.y.dim() == 2 else -1
        if h < 2 or w < 2 or h % 2 or w % 2:
            raise ValueError(f'{what}: frame {i}: an NV12 Y plane must be [h, w] with h and w even, got {list(f.y.shape)}')
        plane(f.y, 'the NV12 Y plane', h, w, 0)
        plane(f.uv, 'the NV12 UV plane', h // 2, w, 0)
    elif isinstance(f, torch.Tensor):
        if f.dim() != 3:
            raise ValueError(f'{what}: frame {i} is {list(f.shape)}; an RGB device frame is uint8 [h, w, 3]')
        plane(f, 'the RGB frame', int(f.shape[0]), int(f.shape[1]), 3)
    else:
        raise ValueError(f'{what}: frame {i} is {type(f).__name__}; a call\'s frames are all numpy arrays or all device frames '
                         '(CUDA tensors, NV12)')


def device_table(frames, plan):
    """Device frames + their FramePlan -> the HOST table (ctypes array of ops.DeviceFrame), checked by
    g6d_frames_table_check: plane pointers, row pitches, size, format and the frame's offset in the packed layout."""
    rows = []
    for f, (off, h, w) in zip(frames, plan.table):
        if isinstance(f, NV12):
            rows.append(ops.DeviceFrame(f.y.data_ptr(), f.uv.data_ptr(), f.y.stride(0) if h > 1 else w, f.uv.stride(0) if h > 2 else w,
                                        h, w, _lib.G6D_FRAME_NV12, off))
        else:
            rows.append(ops.DeviceFrame(f.data_ptr(), None, f.stride(0) if h > 1 else 3 * w, 0, h, w, _lib.G6D_FRAME_RGB, off))
    table = (ops.DeviceFrame * len(rows))(*rows)
    ops.frames_table_check(table, plan.nbytes)
    return table


def resized_table(frames, plan):
    """Device frames, at least one of them Resized, + their FramePlan (of working sizes) -> the HOST table (ctypes array
    of ops.ResizedFrame), checked by g6d_frames_resized_table_check: a plain frame is an identity row (working size =
    source size, no rotation)."""
    rows = []
    for f, (off, _, _) in zip(frames, plan.table):
        (rh, rw), rot, f = (f.size, f.rotate, f.frame) if isinstance(f, Resized) else (f.shape[:2], 0, f)
        h, w = int(f.shape[0]), int(f.shape[1])
        if isinstance(f, NV12):
            rows.append(ops.ResizedFrame(f.y.data_ptr(), f.uv.data_ptr(), f.y.stride(0) if h > 1 else w, f.uv.stride(0) if h > 2 else w,
                                         h, w, _lib.G6D_FRAME_NV12, rh, rw, rot, off))
        else:
            rows.append(ops.ResizedFrame(f.data_ptr(), None, f.stride(0) if h > 1 else 3 * w, 0, h, w, _lib.G6D_FRAME_RGB, rh, rw,
                                         rot, off))
    table = (ops.ResizedFrame * len(rows))(*rows)
    ops.frames_resized_table_check(table, plan.nbytes)
    return table


def check_frames(que_imgs, que_Ks, what):
    """-> the frames as numpy arrays (device frames, checked by as_frames, as they are); ValueError unless there is at
    least one frame, one K per frame and every numpy frame is uint8 [h, w, 3]."""
    if is_device(que_imgs):
        frames = list(que_imgs)
        if not frames or len(que_Ks) != len(frames):
            raise ValueError(f'{what}: {len(frames)} frames and {len(que_Ks)} intrinsics; need one K per frame and at least one frame')
        return frames
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

    def device_key(self, name, resized=False):
        """The graph name of `name` (the numpy path's name of this pattern) for device frames of this size pattern;
        resized: the frames hold a Resized frame (the pattern is of working sizes, and the sources live in the table)."""
        return ('device-resized' if resized else 'device', name, self.pattern)

    def device_upload(self, module, frames, resized=False):
        """Device frames -> graph inputs [table u8 [qn*56]] (one size) or [table, order int64 [qn]] (several): the checked
        g6d_device_frame rows (g6d_resized_frame rows of 64 bytes when resized), uploaded like any small input.  The
        frames themselves are not copied."""
        table = np.frombuffer(bytes(resized_table(frames, self) if resized else device_table(frames, self)), np.uint8)
        return [module._to_dev(table)] + ([module._to_dev(self.order)] if self.mixed else [])

    def gathered(self, fn, resized=False):
        """A graph body fn(frames u8 [qn,h,w,3], *rest) -> g(table, *rest) for device frames: g6d_frames_gather (or, when
        resized, g6d_frames_gather_resized) writes the packed layout from the table, then fn runs on its [qn,h,w,3] view
        (one size) or through on_canvas (several)."""
        qn, (h, w) = len(self.pattern), self.pattern[0]
        body = on_canvas(fn, self) if self.mixed else fn
        gather = ops.frames_gather_resized if resized else ops.frames_gather

        def g(table, *rest):
            packed = gather(table, qn, self.H, self.W, self.nbytes)
            return body(packed, *rest) if self.mixed else body(packed[:qn * h * w * 3].view(qn, h, w, 3), *rest)
        return g


def bind(module, name, fn, frames, plan):
    """A graph name as the numpy path names it (the pattern's key for several sizes), its body fn(frames u8 [qn,h,w,3],
    *rest) and the frames -> (graph name, graph body, frame inputs) for StageCache.run(name, body, frame inputs + rest).
    Numpy frames of one size: (name, fn, [the frames uploaded as [qn,h,w,3]]), exactly the single-size path; of several:
    on_canvas(fn) and the packed upload; device frames: the pattern's device key, the gather body and the table (the
    'device-resized' key, the resized gather and its table when a frame is Resized, row f15)."""
    if is_device(frames):
        r = has_resized(frames)
        return plan.device_key(name, r), plan.gathered(fn, r), plan.device_upload(module, frames, r)
    if not plan.mixed:
        return name, fn, [module.upload_frame(frames)]
    return name, on_canvas(fn, plan), plan.upload(module, frames)


def stage(module, name, fn, frames, plan=None):
    """A graph body fn(frames u8 [qn,h,w,3], *rest) and the frames (numpy, or device frames from as_frames) -> (graph
    name, graph body, frame inputs) for StageCache.run(name, fn, frame inputs + rest).  Numpy frames of one size: (name,
    fn, [the frames uploaded as [qn,h,w,3]]), exactly the single-size path; several: the pattern's name, on_canvas(fn)
    and the packed upload; device frames: bind's device graph."""
    plan = plan or FramePlan(size_pattern(frames))
    return bind(module, plan.key(name) if plan.mixed else name, fn, frames, plan)


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
