"""Common plumbing of the three network classes: lazily packed weights and numpy <-> device IO."""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..graphs import StageCache


IO_BYTES = {'h2d': 0, 'd2h': 0}   # bytes moved through the numpy-facing API (bench.py reads this)


class PackedModule(nn.Module):
    """nn.Module whose parameters are re-packed for the kernels on first use and whenever the
    parameters change (load_state_dict, .cuda(), .to())."""

    def __init__(self):
        super().__init__()
        self._packed = None
        self.stages = StageCache()      # CUDA graphs of the fixed-shape numpy-API stages
        self._pinned, self._pinned_next = {}, {}
        self.generation = 0             # bumped whenever weights or cached reference state change (worker clones go stale)
        self.weights_generation = 0     # bumped whenever the weights change (reference state computed with them goes stale)
        self.register_load_state_dict_post_hook(lambda module, keys: module.invalidate_packed())

    def bump_generation(self):
        """Called after anything a worker_clone() shares by reference was replaced: packed weights,
        cached reference features.  Holders of clones (Gen6DEstimator.predict_many) compare it."""
        self.generation += 1
        self.stages.clear()             # captured graphs hold pointers into the previous state

    def invalidate_packed(self):
        self._packed = None
        self.weights_generation += 1
        self.bump_generation()

    def _apply(self, fn, *args, **kwargs):
        self._packed = None
        self.weights_generation += 1
        self.bump_generation()
        return super()._apply(fn, *args, **kwargs)

    @property
    def device(self):
        return next(self.parameters()).device

    def packed(self):
        if self._packed is None:
            ops.require_cuda()
            if self.device.type != 'cuda':
                raise RuntimeError(f'{type(self).__name__}: parameters are on {self.device}; call .cuda() first '
                                   '(the Gen6D hot path has no CPU fallback)')
            with torch.no_grad():
                self._packed = self._pack()
        return self._packed

    def _pack(self):
        raise NotImplementedError

    def worker_clone(self):
        """A second handle on the same network for another host thread / CUDA stream: parameters,
        packed weights and cached reference features are shared (read-only on the device); the
        CUDA-graph stages (static buffers) and pinned staging buffers are private."""
        import copy
        self.packed()
        other = copy.copy(self)
        other.stages = StageCache()
        other._pinned, other._pinned_next = {}, {}
        other.__dict__.pop('_s2_done', None)         # per-handle scratch (selector): never shared between streams
        return other

    def _to_dev(self, array, dtype=None):
        """numpy -> device through a cached pinned staging buffer (async H2D on the current stream).
        The host-side copy into the staging buffer is a plain single-threaded numpy copy: torch's
        multi-threaded CPU copy_ turns a 3.7 MB frame batch into a ~40 ms OpenMP barrier stall when several
        host threads drive the GPU under a CPU quota (measured; numpy: 0.3 ms)."""
        parts = None
        if isinstance(array, (list, tuple)) and len(array) and all(isinstance(a, np.ndarray) and a.shape == array[0].shape and
                                                                  a.dtype == array[0].dtype for a in array) and dtype is None:
            # equally shaped arrays (the frames of a batch): copied one by one into the [n, ...] staging buffer,
            # without the intermediate np.stack (a second 9 MB host copy for ten 480x640 frames)
            parts, shape, dt = array, (len(array),) + array[0].shape, array[0].dtype
        else:
            arr = np.ascontiguousarray(array)
            if dtype is not None:
                arr = arr.astype(torch.empty(0, dtype=dtype).numpy().dtype, copy=False)
            shape, dt = arr.shape, arr.dtype
        slot = self._pinned_slot(shape, dt)
        if parts is not None:
            dst = slot.numpy()
            for i, a in enumerate(parts):
                np.copyto(dst[i], a)
        else:
            np.copyto(slot.numpy(), arr)
        IO_BYTES['h2d'] += slot.numel() * slot.element_size()
        return slot.to(self.device, non_blocking=True)

    def _pinned_slot(self, shape, dt):
        """The next of (up to) four pinned staging buffers of this shape and dtype, used round robin."""
        key = (shape, dt.str)
        ring = self._pinned.setdefault(key, [])
        if len(ring) < 4:
            ring.append(torch.from_numpy(np.empty(shape, dt)).pin_memory())
        slot = ring[self._pinned_next.get(key, 0) % len(ring)]
        self._pinned_next[key] = self._pinned_next.get(key, 0) + 1
        return slot

    def upload_packed(self, arrays, offsets, nbytes):
        """uint8 arrays -> one device uint8 buffer [nbytes] holding array i's bytes at offsets[i], through the pinned
        staging of _to_dev (one H2D copy).  Bytes no array covers are zero."""
        slot = self._pinned_slot((int(nbytes),), np.dtype(np.uint8))
        dst = slot.numpy()
        end = 0
        for a, off in zip(arrays, offsets):
            if off > end:
                dst[end:off] = 0
            end = off + a.nbytes
            np.copyto(dst[off:end].reshape(a.shape), a)
        dst[end:] = 0
        IO_BYTES['h2d'] += slot.numel()
        return slot.to(self.device, non_blocking=True)

    def upload_frame(self, que_img):
        """uint8 [h,w,3] query frame (or a list of equally sized frames -> [qn,h,w,3]) -> device, once per
        frame: the detector reads it, the detection crop and every refinement iteration's look-at crop are cut
        from it on the device."""
        return self._to_dev(que_img)

    @staticmethod
    def _to_host(t):
        """device -> numpy (synchronising D2H read of a result)."""
        IO_BYTES['d2h'] += t.numel() * t.element_size()
        return t.cpu().numpy()


class Branches:
    """Fork/join of independent sub-graphs onto side streams (the four detector scales, the three
    selector towers, the refiner's feature branches).  At batch 1 most of their kernels launch far
    fewer CTAs than the GPU has SMs, so running the branches concurrently is what fills the machine.
    Works eagerly and under CUDA-graph capture (the side streams fork from and join back into the
    capturing stream, so the captured graph gets parallel branches).  Branch results must be kept
    alive by the caller until they have been consumed on the main stream.  G6D_BRANCH_STREAMS=0
    serialises everything on the current stream.
    The side streams are pooled per (device, main stream): host threads that drive different main
    streams (predict_many workers) never share a side stream, so concurrent captures cannot fork the
    same stream twice and the caching allocator never hands a block freed under one thread's side
    stream to another thread's work on it."""
    _pool = {}
    _pool_lock = __import__('threading').Lock()

    def __init__(self, n):
        import os
        self.enabled = os.environ.get('G6D_BRANCH_STREAMS', '1') != '0' and n > 1
        self.main = torch.cuda.current_stream()
        if self.enabled:
            key = (torch.cuda.current_device(), self.main.cuda_stream)
            with Branches._pool_lock:
                pool = Branches._pool.setdefault(key, [])
                while len(pool) < n:
                    pool.append(torch.cuda.Stream())
                self.streams = pool[:n]
            for st in self.streams:
                st.wait_stream(self.main)

    def run(self, i, fn):
        if not self.enabled:
            return fn()
        with torch.cuda.stream(self.streams[i]):
            return fn()

    def join(self):
        if self.enabled:
            for st in self.streams:
                self.main.wait_stream(st)


def linear_as_conv(weight, bias, cin_pad=None):
    """nn.Linear / Conv1d(k=1) / Conv2d(k=1) weight -> PackedConv of a 1x1 convolution."""
    w = weight.reshape(weight.shape[0], weight.shape[1], 1)
    return ops.pack_conv(w, bias, stride=1, pad=0, cin_pad=cin_pad)
