"""Boxes from another detector (DESIGN.md row f19): caller-supplied 2-D boxes replace the detector's score maps and peaks.

This module is the only place that knows the box format.  A frame's boxes are a float array or a CUDA float32 tensor
[n, 4] (x0, y0, x1, y1; score 0) or [n, 5] (x0, y0, x1, y1, score), in the frame's own pixels (a frames.Resized frame's
working pixels, after the resize and the rotation); n may be 0.  An object set takes a dict {object name: such boxes}
per frame, a missing name meaning no boxes for that object.

The boxes of a call are packed into one table of maps, map j = o*qn + f being object o on frame f (the map order of
g6d_det_parse_peaks): [n_maps, N, 5] float32 boxes and int32 counts, with N the next power of two of the longest list
(at least 1), so calls with different box counts replay one graph per bucket.  Table and counts travel as one float32
buffer (the counts' int32 bits after the boxes): numpy boxes go up in one copy, CUDA boxes are copied device to device
into it, without a host synchronise.  g6d_det_from_boxes turns the table into detection records inside the graph.
"""
import numpy as np
import torch

from . import _lib, ops


def inv_box_size(ref_resolution):
    """The record's scale factor: float32(1 / ref_resolution), exact for ref_resolution 128."""
    return float(np.float32(1.0 / float(ref_resolution)))


def bucket(n):
    """The table width N for a longest list of n boxes: the next power of two, at least 1."""
    return 1 << max(int(n) - 1, 0).bit_length()


def _parse(b, what, device):
    """One map's boxes -> a float32 [n, 5] numpy array or a CUDA float32 tensor [n, 4|5] on `device`; ValueError for boxes on
    a CPU tensor, another device or dtype, a wrong shape, more than G6D_DET_MAX_BOXES boxes, and numpy boxes that are
    non-finite or degenerate (x1 <= x0 or y1 <= y0).  CUDA boxes are not read here: the kernel skips unusable ones."""
    if isinstance(b, torch.Tensor):
        if not b.is_cuda:
            raise ValueError(f'{what}: boxes on a CPU tensor; pass a numpy array or a CUDA float32 tensor')
        if b.device != torch.device(device):
            raise ValueError(f'{what}: boxes on {b.device}; CUDA boxes must be on {device}, the estimator\'s device')
        if b.dtype != torch.float32:
            raise ValueError(f'{what}: CUDA boxes are {b.dtype}; need float32')
        shape = tuple(b.shape)
    else:
        a = np.asarray(b)
        if a.dtype.kind not in 'fiu':
            raise ValueError(f'{what}: boxes of dtype {a.dtype}; need a float array')
        shape = a.shape
    if len(shape) != 2 or shape[1] not in (4, 5):
        raise ValueError(f'{what}: boxes are {list(shape)}; need [n, 4] (x0, y0, x1, y1) or [n, 5] (x0, y0, x1, y1, score)')
    if shape[0] > _lib.G6D_DET_MAX_BOXES:
        raise ValueError(f'{what}: {shape[0]} boxes on one map; at most {_lib.G6D_DET_MAX_BOXES}')
    if isinstance(b, torch.Tensor):
        return b
    with np.errstate(over='ignore'):
        a = a.astype(np.float32)                             # values past float32's range become inf, rejected below
    if not np.isfinite(a).all():
        raise ValueError(f'{what}: boxes hold non-finite values')
    if ((a[:, 2] <= a[:, 0]) | (a[:, 3] <= a[:, 1])).any():
        raise ValueError(f'{what}: degenerate boxes (need x1 > x0 and y1 > y0)')
    return np.concatenate([a, np.zeros((len(a), 1), np.float32)], 1) if shape[1] == 4 else a


class Table:
    """The parsed boxes of n_maps maps (None: no boxes) -> N, the host counts and upload(): the graph's box buffer."""

    def __init__(self, maps):
        self.maps = maps
        self.n_maps = len(maps)
        self.counts = np.asarray([0 if m is None else int(m.shape[0]) for m in maps], np.int32)
        self.N = bucket(self.counts.max(initial=0))

    def host(self):
        """The numpy maps and counts as the buffer's bytes (CUDA maps left zero)."""
        n, N = self.n_maps, self.N
        buf = np.zeros(n * N * 5 + n, np.float32)
        tab = buf[:n * N * 5].reshape(n, N, 5)
        for j, m in enumerate(self.maps):
            if isinstance(m, np.ndarray) and len(m):
                tab[j, :len(m)] = m
        buf[n * N * 5:] = self.counts.view(np.float32)
        return buf

    def upload(self, module):
        """-> float32 buffer [n_maps*N*5 + n_maps] on module's device: one copy of the host part, then every CUDA map
        copied into its rows on the current stream."""
        buf = module._to_dev(self.host())
        tab = split(buf, self.n_maps, self.N)[0]
        for j, m in enumerate(self.maps):
            if isinstance(m, torch.Tensor) and m.shape[0]:
                tab[j, :m.shape[0], :m.shape[1]].copy_(m)
        return buf


def split(buf, n_maps, N):
    """The box buffer -> (boxes float32 [n_maps, N, 5], counts int32 [n_maps]), views."""
    return buf[:n_maps * N * 5].view(n_maps, N, 5), buf[n_maps * N * 5:].view(torch.int32)


def host_records(boxes, counts, max_inst, inv):
    """g6d_det_from_boxes_host on numpy arrays: boxes [n_maps, N, 5], counts [n_maps] -> (det float32 [max_inst, n_maps, 4],
    valid int32 [max_inst, n_maps], count int32 [n_maps]), the device kernel's bytes."""
    boxes, counts = np.ascontiguousarray(boxes, np.float32), np.ascontiguousarray(counts, np.int32)
    n, N, _ = boxes.shape
    det = np.zeros((max_inst, n, 4), np.float32)
    valid, count = np.zeros((max_inst, n), np.int32), np.zeros(n, np.int32)
    _lib.check(_lib.lib().g6d_det_from_boxes_host(boxes.ctypes.data, counts.ctypes.data, n, N, int(max_inst), float(inv),
                                                  det.ctypes.data, valid.ctypes.data, count.ctypes.data), 'g6d_det_from_boxes_host')
    return det, valid, count


def check_len(boxes, n, what, of):
    """ValueError unless boxes holds one entry per `of` (n of them)."""
    if boxes is None or isinstance(boxes, (dict, str)) or len(boxes) != n:
        got = 'None' if boxes is None else type(boxes).__name__ if isinstance(boxes, (dict, str)) else f'{len(boxes)} entries'
        raise ValueError(f'{what}: boxes needs one entry per {of} ({n}), got {got}')


def for_frames(boxes, qn, what, device):
    """An estimator call's boxes, one array per frame -> Table (map j = frame j)."""
    check_len(boxes, qn, what, 'frame')
    return Table([_parse(b, f'{what}: frame {f}', device) for f, b in enumerate(boxes)])


def one_per_frame(boxes, qn, what):
    """predict_batch's boxes, exactly one per frame ([4], [5] or [1, 4|5]) -> a [1, 4|5] list per frame, as for_frames
    takes them."""
    check_len(boxes, qn, what, 'frame')
    out = []
    for f, b in enumerate(boxes):
        shape = tuple(b.shape) if isinstance(b, torch.Tensor) else np.shape(b)
        if shape not in ((4,), (5,), (1, 4), (1, 5)):
            raise ValueError(f'{what}: frame {f}: box is {list(shape)}; need exactly one box per frame: [4], [5] or [1, 4|5]')
        out.append(b.reshape(1, -1) if isinstance(b, torch.Tensor) else np.reshape(b, (1, -1)))
    return out


def _object_maps(entries, names, what, device):
    """Per frame a dict {name: boxes} (or None: no boxes) -> the maps o*n + f of the frames' objects."""
    n, maps = len(entries), [None] * (len(names) * len(entries))
    for f, d in enumerate(entries):
        if d is None:
            continue
        if not isinstance(d, dict):
            raise ValueError(f'{what}: entry {f} is {type(d).__name__}; an object set takes a dict {{object name: boxes}} per frame')
        unknown = [k for k in d if k not in names]
        if unknown:
            raise ValueError(f'{what}: entry {f} names objects {unknown} that are not in the set (objects: {list(names)})')
        for o, name in enumerate(names):
            if name in d:
                maps[o * n + f] = _parse(d[name], f'{what}: entry {f}, object {name!r}', device)
    return maps


def for_objects(boxes, names, qn, what, device):
    """An object set call's boxes, a dict {name: boxes} per frame -> Table (map j = o*qn + f)."""
    check_len(boxes, qn, what, 'frame')
    return Table(_object_maps(list(boxes), names, what, device))


def for_sequences(boxes, n, what, device, names=None):
    """A tracker step's boxes, one entry per stepped sequence (None: no boxes for it) -> (Table, has bool [n]): the
    sequences given boxes.  names: an object set's objects (dict entries), None: the estimator's (array entries)."""
    check_len(boxes, n, what, 'stepped sequence')
    entries = list(boxes)
    has = np.asarray([e is not None for e in entries], bool)
    if names is not None:
        return Table(_object_maps(entries, names, what, device)), has
    return Table([None if e is None else _parse(e, f'{what}: sequence entry {s}', device) for s, e in enumerate(entries)]), has


def graph_name(base, N):
    """The graph name of a box body: apart from every detector-path name, keyed on the table width N."""
    return ('boxes', N, base)


class Detect:
    """The detection step of a box graph: detect(frames) -> det [M*n_maps, 4] instance-major, with .extra = [valid int32
    [M*n_maps], count int32 [n_maps]] once it ran.  bind(fn) makes a graph body that takes the box buffer as its last input;
    select(seq) (a mixed tracker step) detects the maps of the gathered frames seq of each of the K objects."""

    def __init__(self, M, K, n_maps, N, inv):
        self.M, self.K, self.n_maps, self.N, self.inv = M, K, n_maps, N, inv
        self.extra, self.buf, self.seq = [], None, None

    def bind(self, fn):
        def g(*args):
            self.buf, self.seq = args[-1], None
            return fn(*args[:-1])
        return g

    def select(self, seq):
        self.seq = seq

    def __call__(self, frames):
        boxes, counts = split(self.buf, self.n_maps, self.N)
        if self.seq is not None:
            b = self.n_maps // self.K
            rows = (torch.arange(self.K, device=self.seq.device, dtype=torch.int64)[:, None] * b + self.seq[None, :]).reshape(-1)
            boxes, counts = boxes.index_select(0, rows), counts.index_select(0, rows)
        det, valid, count = ops.det_from_boxes(boxes, counts, self.M, self.inv)
        self.extra[:] = [valid.reshape(-1), count]
        return det.reshape(-1, 4)
