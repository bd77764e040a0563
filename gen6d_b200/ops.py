"""Torch-tensor front end of the C ABI.

PyTorch is used here only as the device-memory allocator and stream provider: every function
checks its tensors (CUDA, contiguous, dtype), takes raw pointers and calls into
libgen6d_b200.so on torch's current stream.  Activations are fp32 channels-last.
"""
import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import ACT_LEAKY01, ACT_NONE, ACT_RELU, PRO_AFFINE, PRO_AFFINE_RELU, PRO_CORR, PRO_NONE  # noqa: F401


WARP_JOB_BYTES = 88   # sizeof(g6d_warp_job)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t, dtype=torch.float32):
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise ValueError(f'expected a contiguous CUDA {dtype} tensor, got {t.dtype} {t.device} '
                         f'contiguous={t.is_contiguous()} shape={tuple(t.shape)}')
    return C.c_void_p(t.data_ptr())


_PROFILE = None   # when enabled: {name: [(start_event, end_event, work), ...]}


def _call(name, *args, work=None, tag=None, key=None):
    """key: the profile entry the call is timed under (default: name)."""
    if _PROFILE is not None and work is not None:
        key = key or name
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(getattr(_lib.lib(), name)(*args), name)
        e1.record()
        _PROFILE.setdefault(key, []).append((e0, e1, work))
        if tag is not None:
            _PROFILE.setdefault('#calls', []).append((e0, e1, work, key, tag))
        return
    _lib.check(getattr(_lib.lib(), name)(*args), name)


def enable_profiling():
    """Time every launch of the roofline kernels with CUDA events on the launching stream
    (bench.py).  `work` is the algorithmic FLOPs (conv) or bytes (streaming kernels) of the call."""
    global _PROFILE
    _PROFILE = {}
    return _PROFILE


def collect_profile(prof):
    global _PROFILE
    torch.cuda.synchronize()
    _PROFILE = None
    out = {k: {'ms': sum(r[0].elapsed_time(r[1]) for r in v), 'work': float(sum(r[2] for r in v)), 'n': len(v)}
           for k, v in prof.items() if k != '#calls'}
    if '#calls' in prof:
        out['#calls'] = [(r[0].elapsed_time(r[1]), r[2], r[3], r[4]() if callable(r[4]) else r[4]) for r in prof['#calls']]
    return out


def require_cuda():
    if not torch.cuda.is_available():
        raise _lib.Gen6DLibraryError('no CUDA device: the Gen6D hot path has no CPU fallback')
    _lib.lib()


# ------------------------------------------------------------------------------- layout / images
def preprocess_u8(img, out_c=4, imagenet_norm=True):
    """u8 [..., H, W, 3] -> f32 [..., H, W, out_c]: /255 (+ ImageNet normalisation)."""
    out = torch.empty(*img.shape[:-1], out_c, device=img.device, dtype=torch.float32)
    _call('g6d_preprocess_u8', _p(img, torch.uint8), _p(out), img.numel() // 3, out_c, int(imagenet_norm), _stream())
    return out


def _warp(name, jobs, n_jobs, h, w):
    if jobs.dtype != torch.uint8 or jobs.numel() != n_jobs * WARP_JOB_BYTES:
        raise ValueError(f'{name}: jobs must be the packed bytes of {n_jobs} g6d_warp_job records')
    out = torch.empty(n_jobs, h, w, 3, device=jobs.device, dtype=torch.uint8)
    _call(name, _p(jobs, torch.uint8), n_jobs, _p(out, torch.uint8), h, w, _stream())
    return out


def warp_perspective_u8(jobs, n_jobs, h, w):
    """cv2.warpPerspective (u8, INTER_LINEAR, zero border), bit-exact, for n_jobs (image, H) pairs.
    jobs: device uint8 tensor holding n_jobs packed g6d_warp_job records (geometry.pack_warp_jobs)."""
    return _warp('g6d_warp_perspective_u8', jobs, n_jobs, h, w)


def warp_affine_u8(jobs, n_jobs, h, w):
    """cv2.warpAffine counterpart of warp_perspective_u8."""
    return _warp('g6d_warp_affine_u8', jobs, n_jobs, h, w)


class FrameEntry(C.Structure):        # g6d_frame_entry
    _fields_ = [('offset', C.c_longlong), ('rows', C.c_int), ('cols', C.c_int)]


def frames_canvas(packed, table, H, W):
    """packed u8 (frames back to back) + table [(byte offset, rows, cols)] per frame (host) -> canvas u8 [n,H,W,3]: every
    frame in the top-left corner, zeros elsewhere (g6d_frames_canvas)."""
    n = len(table)
    if packed.dtype != torch.uint8 or packed.dim() != 1:
        raise ValueError('frames_canvas: packed must be a 1-D uint8 tensor')
    host = (FrameEntry * max(n, 1))(*[FrameEntry(int(o), int(r), int(c)) for o, r, c in table])
    out = torch.empty(n, H, W, 3, device=packed.device, dtype=torch.uint8)
    _call('g6d_frames_canvas', _p(packed, torch.uint8), packed.numel(), host, n, _p(out, torch.uint8) if n else None, H, W,
          _stream())
    return out


class DeviceFrame(C.Structure):       # g6d_device_frame
    _fields_ = [('plane0', C.c_void_p), ('plane1', C.c_void_p), ('pitch0', C.c_longlong), ('pitch1', C.c_longlong),
                ('rows', C.c_int), ('cols', C.c_int), ('format', C.c_int), ('offset', C.c_longlong)]


def frames_table_check(table, nbytes):
    """A HOST array of DeviceFrame (ctypes) -> None; Gen6DLibraryError (G6D_EINVAL, with the message) unless every entry
    is valid for a packed buffer of nbytes bytes (g6d_frames_table_check)."""
    _call('g6d_frames_table_check', table, len(table), int(nbytes))


def frames_gather(table, n, max_rows, max_cols, nbytes):
    """table: the bytes of n DeviceFrame entries on the device (uint8 [n*sizeof]) -> packed u8 [nbytes]: every frame's RGB
    image at its offset, 0 elsewhere (g6d_frames_gather)."""
    if table.dtype != torch.uint8 or table.numel() != n * C.sizeof(DeviceFrame):
        raise ValueError(f'frames_gather: table must be the packed bytes of {n} g6d_device_frame records')
    out = torch.empty(int(nbytes), device=table.device, dtype=torch.uint8)
    _call('g6d_frames_gather', _p(table, torch.uint8), n, max_rows, max_cols, _p(out, torch.uint8), int(nbytes), _stream())
    return out


def frames_gather_host(table, nbytes):
    """g6d_frames_gather on the host: a HOST array of DeviceFrame over host planes -> numpy u8 [nbytes]."""
    import numpy as np
    out = np.empty(int(nbytes), np.uint8)
    _call('g6d_frames_gather_host', table, len(table), out.ctypes.data_as(C.c_void_p), int(nbytes))
    return out


class ResizedFrame(C.Structure):      # g6d_resized_frame
    _fields_ = [('plane0', C.c_void_p), ('plane1', C.c_void_p), ('pitch0', C.c_longlong), ('pitch1', C.c_longlong),
                ('src_rows', C.c_int), ('src_cols', C.c_int), ('format', C.c_int), ('rows', C.c_int), ('cols', C.c_int),
                ('rotate', C.c_int), ('offset', C.c_longlong)]


def frames_resized_table_check(table, nbytes):
    """A HOST array of ResizedFrame (ctypes) -> None; Gen6DLibraryError (G6D_EINVAL, with the message) unless every entry
    is valid for a packed buffer of nbytes bytes (g6d_frames_resized_table_check)."""
    _call('g6d_frames_resized_table_check', table, len(table), int(nbytes))


def frames_gather_resized(table, n, max_rows, max_cols, nbytes):
    """table: the bytes of n ResizedFrame entries on the device (uint8 [n*sizeof]) -> packed u8 [nbytes]: every frame's
    resized, rotated RGB image at its offset, 0 elsewhere (g6d_frames_gather_resized).  max_rows / max_cols bound the
    working (rotated) sizes."""
    if table.dtype != torch.uint8 or table.numel() != n * C.sizeof(ResizedFrame):
        raise ValueError(f'frames_gather_resized: table must be the packed bytes of {n} g6d_resized_frame records')
    out = torch.empty(int(nbytes), device=table.device, dtype=torch.uint8)
    _call('g6d_frames_gather_resized', _p(table, torch.uint8), n, max_rows, max_cols, _p(out, torch.uint8), int(nbytes),
          _stream())
    return out


def frames_gather_resized_host(table, nbytes):
    """g6d_frames_gather_resized on the host: a HOST array of ResizedFrame over host planes -> numpy u8 [nbytes]."""
    import numpy as np
    out = np.empty(int(nbytes), np.uint8)
    _call('g6d_frames_gather_resized_host', table, len(table), out.ctypes.data_as(C.c_void_p), int(nbytes))
    return out


# ------------------------------------------------------------------------------- camera algebra between the stages
def glue_detection_jobs(det_out, frames, size):
    """det_out [qn,4] (g6d_det_parse) + frames u8 [qn,h,w,3] -> packed g6d_warp_job records [qn*88] of the selector crops."""
    qn, h, w, _ = frames.shape
    jobs = torch.empty(qn * WARP_JOB_BYTES, device=frames.device, dtype=torch.uint8)
    _call('g6d_glue_detection_jobs', _p(det_out), _p(frames, torch.uint8), h, w, qn, size, _p(jobs, torch.uint8), _stream())
    return jobs


def glue_initial_poses(det_out, sel_idx, sel_out, refs_struct, cams):
    """Detection + selection -> initial poses float64 [qn,12] (geometry.poses_from_similarity on the device)."""
    qn = det_out.shape[0]
    poses = torch.empty(qn, 12, device=det_out.device, dtype=torch.float64)
    _call('g6d_glue_initial_poses', _p(det_out), _p(sel_idx, torch.int64), _p(sel_out), C.byref(refs_struct), _p(cams, torch.float64),
          qn, _p(poses, torch.float64), _stream())
    return poses


def glue_refine_problems(views_struct, ref_num, cams, frames, poses, poses_are_f32):
    """poses float64 [qn,12] -> (jobs u8 [qn*(ref_num+1)*88], que_K [qn,3,3], que_pose [qn,3,4], rect [qn,3,4],
    ref_Ks [qn,R,3,3], ref_poses [qn,R,3,4], ref_rows i32 [qn,R]): geometry.refine_problems on the device."""
    qn, h, w, _ = frames.shape
    dev, f32 = frames.device, torch.float32
    jobs = torch.empty(qn * (ref_num + 1) * WARP_JOB_BYTES, device=dev, dtype=torch.uint8)
    que_K, que_pose, rect = torch.empty(qn, 3, 3, device=dev, dtype=f32), torch.empty(qn, 3, 4, device=dev, dtype=f32), \
        torch.empty(qn, 3, 4, device=dev, dtype=f32)
    ref_Ks, ref_poses = torch.empty(qn, ref_num, 3, 3, device=dev, dtype=f32), torch.empty(qn, ref_num, 3, 4, device=dev, dtype=f32)
    rows = torch.empty(qn, ref_num, device=dev, dtype=torch.int32)
    _call('g6d_glue_refine_problems', C.byref(views_struct), _p(cams, torch.float64), _p(frames, torch.uint8), h, w,
          _p(poses, torch.float64), int(poses_are_f32), qn, _p(jobs, torch.uint8), _p(que_K), _p(que_pose), _p(rect), _p(ref_Ks),
          _p(ref_poses), _p(rows, torch.int32), _stream())
    return jobs, que_K, que_pose, rect, ref_Ks, ref_poses, rows


def glue_apply_refinements(views_struct, que_pose, que_K, rect, net_out):
    """Network output [qn,7] -> refined poses (float32 values) float64 [qn,12]: geometry.apply_refinements on the device."""
    qn = net_out.shape[0]
    poses = torch.empty(qn, 12, device=net_out.device, dtype=torch.float64)
    _call('g6d_glue_apply_refinements', C.byref(views_struct), _p(que_pose), _p(que_K), _p(rect), _p(net_out), qn,
          _p(poses, torch.float64), _stream())
    return poses


def _object_chunks(n_obj):
    """Object ranges of the g6d_glue_*_objects launches (their view structs travel as one kernel parameter block)."""
    step = _lib.G6D_GLUE_MAX_OBJECTS
    return [(o, min(o + step, n_obj)) for o in range(0, n_obj, step)]


def _views_array(views_structs, o0, o1):
    return (_lib.GlueViews * (o1 - o0))(*views_structs[o0:o1])


def glue_refine_problems_objects(views_structs, ref_num, cams, frames, poses, poses_are_f32):
    """glue_refine_problems for K objects on the same qn frames: poses float64 [K*qn,12], object-major (row o*qn + s is
    object o on frame s, with views_structs[o]) -> the per-object results concatenated along the rows, in one launch
    per G6D_GLUE_MAX_OBJECTS objects."""
    qn, h, w, _ = frames.shape
    K = len(views_structs)
    n = K * qn
    if poses.shape != (n, 12):
        raise ValueError(f'glue_refine_problems_objects: poses {tuple(poses.shape)} for {K} objects x {qn} frames')
    dev, f32 = frames.device, torch.float32
    jobs = torch.empty(n, (ref_num + 1) * WARP_JOB_BYTES, device=dev, dtype=torch.uint8)
    que_K, que_pose, rect = torch.empty(n, 3, 3, device=dev, dtype=f32), torch.empty(n, 3, 4, device=dev, dtype=f32), \
        torch.empty(n, 3, 4, device=dev, dtype=f32)
    ref_Ks, ref_poses = torch.empty(n, ref_num, 3, 3, device=dev, dtype=f32), torch.empty(n, ref_num, 3, 4, device=dev, dtype=f32)
    rows = torch.empty(n, ref_num, device=dev, dtype=torch.int32)
    for o0, o1 in _object_chunks(K):
        r = slice(o0 * qn, o1 * qn)
        _call('g6d_glue_refine_problems_objects', _views_array(views_structs, o0, o1), o1 - o0, qn, _p(cams, torch.float64),
              _p(frames, torch.uint8), h, w, _p(poses[r], torch.float64), int(poses_are_f32), _p(jobs[r], torch.uint8), _p(que_K[r]),
              _p(que_pose[r]), _p(rect[r]), _p(ref_Ks[r]), _p(ref_poses[r]), _p(rows[r], torch.int32), _stream())
    return jobs.reshape(-1), que_K, que_pose, rect, ref_Ks, ref_poses, rows


def glue_apply_refinements_objects(views_structs, que_pose, que_K, rect, net_out):
    """glue_apply_refinements for K objects, rows object-major (K*qn rows, row o*qn + s with views_structs[o]) ->
    refined poses float64 [K*qn,12], in one launch per G6D_GLUE_MAX_OBJECTS objects."""
    K, n = len(views_structs), net_out.shape[0]
    if n % K:
        raise ValueError(f'glue_apply_refinements_objects: {n} rows for {K} objects')
    qn = n // K
    poses = torch.empty(n, 12, device=net_out.device, dtype=torch.float64)
    for o0, o1 in _object_chunks(K):
        r = slice(o0 * qn, o1 * qn)
        _call('g6d_glue_apply_refinements_objects', _views_array(views_structs, o0, o1), o1 - o0, qn, _p(que_pose[r]), _p(que_K[r]),
              _p(rect[r]), _p(net_out[r]), _p(poses[r], torch.float64), _stream())
    return poses


def _row_chunks(views_structs, rows_per_obj, row_idx):
    """(o0, o1, list slice, row indices relative to object o0) per G6D_GLUE_MAX_OBJECTS objects: the list is object-major
    with the same number of entries per object, so it splits at static offsets."""
    K, n_sel = len(views_structs), row_idx.shape[0]
    if n_sel < 1 or n_sel % K:
        raise ValueError(f'glue rows: {n_sel} listed rows for {K} objects; every object lists the same number of rows')
    per = n_sel // K
    out = []
    for o0, o1 in _object_chunks(K):
        r = slice(o0 * per, o1 * per)
        idx = row_idx[r] if o0 == 0 else (row_idx[r] - o0 * rows_per_obj).contiguous()
        out.append((o0, o1, r, idx))
    return out


def glue_refine_problems_rows(views_structs, ref_num, rows_per_obj, cams, frames, poses, row_idx, row_f32):
    """glue_refine_problems_objects on the listed rows only: poses float64 [K*rows_per_obj,12] (object-major, row o*rows_per_obj
    + s is object o on frame s), row_idx int32 [n_sel] (object-major, the same count per object), row_f32 uint8
    [K*rows_per_obj] (each row's dtype flag) -> the problems of the listed rows, output row j being row row_idx[j]."""
    qn, h, w, _ = frames.shape
    K, n_sel = len(views_structs), row_idx.shape[0]
    n = K * rows_per_obj
    if poses.shape != (n, 12) or row_f32.shape != (n,) or qn != rows_per_obj or cams.shape[0] != rows_per_obj:
        raise ValueError(f'glue_refine_problems_rows: poses {tuple(poses.shape)}, row_f32 {tuple(row_f32.shape)}, frames {qn}, '
                         f'cams {cams.shape[0]} for {K} objects x {rows_per_obj} rows')
    dev, f32 = frames.device, torch.float32
    jobs = torch.empty(n_sel, (ref_num + 1) * WARP_JOB_BYTES, device=dev, dtype=torch.uint8)
    que_K, que_pose, rect = torch.empty(n_sel, 3, 3, device=dev, dtype=f32), torch.empty(n_sel, 3, 4, device=dev, dtype=f32), \
        torch.empty(n_sel, 3, 4, device=dev, dtype=f32)
    ref_Ks, ref_poses = torch.empty(n_sel, ref_num, 3, 3, device=dev, dtype=f32), torch.empty(n_sel, ref_num, 3, 4, device=dev, dtype=f32)
    rows = torch.empty(n_sel, ref_num, device=dev, dtype=torch.int32)
    for o0, o1, r, idx in _row_chunks(views_structs, rows_per_obj, row_idx):
        p = slice(o0 * rows_per_obj, o1 * rows_per_obj)
        _call('g6d_glue_refine_problems_rows', _views_array(views_structs, o0, o1), o1 - o0, rows_per_obj, _p(cams, torch.float64),
              _p(frames, torch.uint8), h, w, _p(poses[p], torch.float64), _p(idx, torch.int32), idx.shape[0], _p(row_f32[p], torch.uint8),
              _p(jobs[r], torch.uint8), _p(que_K[r]), _p(que_pose[r]), _p(rect[r]), _p(ref_Ks[r]), _p(ref_poses[r]),
              _p(rows[r], torch.int32), _stream())
    return jobs.reshape(-1), que_K, que_pose, rect, ref_Ks, ref_poses, rows


def glue_apply_refinements_rows(views_structs, rows_per_obj, que_pose, que_K, rect, net_out, row_idx, poses):
    """glue_apply_refinements_objects for the rows of glue_refine_problems_rows: network output row j updates
    poses[row_idx[j]] (float64 [K*rows_per_obj,12]) in place; the other rows are untouched.  Returns poses."""
    K = len(views_structs)
    if poses.shape != (K * rows_per_obj, 12) or net_out.shape[0] != row_idx.shape[0]:
        raise ValueError(f'glue_apply_refinements_rows: poses {tuple(poses.shape)}, {net_out.shape[0]} outputs for {row_idx.shape[0]} '
                         f'rows, {K} objects x {rows_per_obj} rows')
    for o0, o1, r, idx in _row_chunks(views_structs, rows_per_obj, row_idx):
        p = slice(o0 * rows_per_obj, o1 * rows_per_obj)
        _call('g6d_glue_apply_refinements_rows', _views_array(views_structs, o0, o1), o1 - o0, rows_per_obj, _p(que_pose[r]), _p(que_K[r]),
              _p(rect[r]), _p(net_out[r]), _p(idx, torch.int32), idx.shape[0], _p(poses[p], torch.float64), _stream())
    return poses


def verify_windows(refs_structs, cams, poses, poses_are_f32):
    """K objects' poses float64 [K*qn,12] (object-major, row o*qn + s with refs_structs[o] and cams[s]) -> the detection
    windows' records float32 [K*qn,4] (cx, cy, s, valid; g6d_verify_windows), one launch per G6D_GLUE_MAX_OBJECTS objects."""
    K, qn = len(refs_structs), cams.shape[0]
    if poses.shape != (K * qn, 12):
        raise ValueError(f'verify_windows: poses {tuple(poses.shape)} for {K} objects x {qn} frames')
    rec = torch.empty(K * qn, 4, device=poses.device, dtype=torch.float32)
    for o0, o1 in _object_chunks(K):
        r = slice(o0 * qn, o1 * qn)
        refs = (_lib.GlueRefs * (o1 - o0))(*refs_structs[o0:o1])
        _call('g6d_verify_windows', _p(poses[r], torch.float64), int(poses_are_f32), refs, o1 - o0, qn, _p(cams, torch.float64),
              _p(rec[r]), _stream())
    return rec


def verify_judge(rec, det, window, ref_resolution, lost_score=None, lost_gate=None):
    """Window records [n,4] + the detector's records on the windows [n,4] -> (out float32 [n,5] = x, y, scale, score,
    offset in the frame; lost int32 [n]) (g6d_verify_judge).  A threshold of None is not applied."""
    n = rec.shape[0]
    out = torch.empty(n, 5, device=rec.device, dtype=torch.float32)
    lost = torch.empty(n, device=rec.device, dtype=torch.int32)
    _call('g6d_verify_judge', _p(rec), _p(det), n, int(window), float(ref_resolution), int(lost_score is not None),
          float(lost_score or 0.0), int(lost_gate is not None), float(lost_gate or 0.0), _p(out), _p(lost, torch.int32), _stream())
    return out, lost


class DrawSrc(C.Structure):           # g6d_draw_src
    _fields_ = [('offset', C.c_longlong), ('pitch', C.c_longlong), ('rows', C.c_int), ('cols', C.c_int)]


class DrawBox(C.Structure):           # g6d_draw_box
    _fields_ = [('dst', C.c_int), ('pose', C.c_int), ('K', C.c_int), ('bbox', C.c_int), ('pose_f32', C.c_int), ('valid', C.c_int),
                ('color', C.c_uint8 * 4)]


def draw_check(srcs, boxes, dsts, n_poses, n_Ks, n_bboxes, n_ids=0):
    """HOST ctypes arrays of DrawSrc, DrawBox and DeviceFrame -> None; Gen6DLibraryError unless they are valid for arrays of
    n_poses poses, n_Ks intrinsics, n_bboxes boxes and n_ids track ids (g6d_draw_check)."""
    _call('g6d_draw_check', srcs, len(srcs), boxes, len(boxes), dsts, len(dsts), int(n_poses), int(n_Ks), int(n_bboxes), int(n_ids))


def draw_boxes(src, srcs, n_src, poses, Ks, bboxes, boxes, n_boxes, dsts, n_dst, max_rows, max_cols, ids=None):
    """predict.py's draw_bbox_3d into every destination (g6d_draw_boxes): src the device address the source frames are
    offset from (srcs: n_src DrawSrc rows on the device), poses float64 [n,12], Ks float64 [m,9], bboxes
    float32 [k,8,3], boxes n_boxes DrawBox rows and dsts n_dst DeviceFrame rows on the device (checked by draw_check); ids:
    int64 track ids a box with valid >= 0 reads (drawn when ids[valid] >= 0)."""
    for t, n, cls in ((srcs, n_src, DrawSrc), (boxes, n_boxes, DrawBox), (dsts, n_dst, DeviceFrame)):
        if t.dtype != torch.uint8 or t.numel() != n * C.sizeof(cls):
            raise ValueError(f'draw_boxes: a table of {n} {cls.__name__} rows must be uint8 [{n * C.sizeof(cls)}]')
    _call('g6d_draw_boxes', C.c_void_p(int(src)), _p(srcs, torch.uint8), n_src, _p(poses, torch.float64), _p(Ks, torch.float64),
          _p(bboxes), _p(ids, torch.int64), _p(boxes, torch.uint8) if n_boxes else None, n_boxes, _p(dsts, torch.uint8), n_dst, max_rows, max_cols, _stream())


def rgb_to_nv12(rgb, y, uv):
    """cv2.cvtColor(rgb, COLOR_RGB2YUV_I420) with U and V interleaved, into the planes y uint8 [h,w] and uv [h/2,w] (any
    row pitches; g6d_rgb_to_nv12): rgb a CUDA uint8 [h,w,3] tensor with unit column steps, h and w even."""
    h, w = int(rgb.shape[0]), int(rgb.shape[1])
    if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3 or rgb.stride(2) != 1 or rgb.stride(1) != 3:
        raise ValueError(f'rgb_to_nv12: rgb must be uint8 [h,w,3] with unit column steps, got {rgb.dtype} {list(rgb.shape)}')
    if tuple(y.shape) != (h, w) or tuple(uv.shape) != (h // 2, w) or y.stride(1) != 1 or uv.stride(1) != 1:
        raise ValueError(f'rgb_to_nv12: planes {list(y.shape)} and {list(uv.shape)} for a {h} x {w} frame')
    if not (rgb.is_cuda and y.is_cuda and uv.is_cuda and y.dtype == uv.dtype == torch.uint8):
        raise ValueError('rgb_to_nv12: rgb, y and uv must be CUDA uint8 tensors')
    _call('g6d_rgb_to_nv12', C.c_void_p(rgb.data_ptr()), rgb.stride(0), h, w, C.c_void_p(y.data_ptr()), y.stride(0),
          C.c_void_p(uv.data_ptr()), uv.stride(0), _stream())


def track_smooth_objects(poses, poses_are_f32, bboxes, Ks, ring, count, weights):
    """track_smooth for K objects through S sequences in one launch, rows object-major: poses float64 [K*S,12] (row o*S + s
    is object o on sequence s), bboxes float32 [K,8,3], Ks float64 [S,9], ring float32 [K*S,num,8,2] and count int32 [K*S]
    (updated in place), weights float64 [num] -> (smoothed float64 [K*S,12], averaged corners float64 [K*S,8,2])."""
    K, S, n, num = bboxes.shape[0], Ks.shape[0], poses.shape[0], ring.shape[1]
    if (bboxes.shape != (K, 8, 3) or Ks.shape != (S, 9) or n != K * S or ring.shape != (n, num, 8, 2) or count.shape != (n,)
            or weights.shape != (num,)):
        raise ValueError(f'track_smooth_objects: inconsistent shapes poses {tuple(poses.shape)}, bboxes {tuple(bboxes.shape)}, '
                         f'Ks {tuple(Ks.shape)}, ring {tuple(ring.shape)}, count {tuple(count.shape)}, weights {tuple(weights.shape)}')
    smoothed = torch.empty(n, 12, device=poses.device, dtype=torch.float64)
    avg = torch.empty(n, 8, 2, device=poses.device, dtype=torch.float64)
    _call('g6d_track_smooth_objects', _p(poses, torch.float64), int(poses_are_f32), _p(bboxes), K, S, _p(Ks, torch.float64), _p(ring),
          _p(count, torch.int32), num, _p(weights, torch.float64), _p(smoothed, torch.float64), _p(avg, torch.float64), _stream())
    return smoothed, avg


def track_smooth(poses, poses_are_f32, bbox, Ks, ring, count, weights):
    """One smoothing step for S tracked sequences (g6d_track_smooth): poses float64 [S,12] (raw), bbox float32 [8,3],
    Ks float64 [S,9], ring float32 [S,num,8,2] and count int32 [S] (updated in place), weights float64 [num] ->
    (smoothed poses float64 [S,12], averaged corners float64 [S,8,2])."""
    S, num = poses.shape[0], ring.shape[1]
    if ring.shape != (S, num, 8, 2) or count.shape != (S,) or weights.shape != (num,) or bbox.shape != (8, 3):
        raise ValueError(f'track_smooth: inconsistent shapes ring {tuple(ring.shape)}, count {tuple(count.shape)}, '
                         f'weights {tuple(weights.shape)}, bbox {tuple(bbox.shape)} for {S} sequences')
    smoothed = torch.empty(S, 12, device=poses.device, dtype=torch.float64)
    avg = torch.empty(S, 8, 2, device=poses.device, dtype=torch.float64)
    _call('g6d_track_smooth', _p(poses, torch.float64), int(poses_are_f32), _p(bbox), _p(Ks, torch.float64), _p(ring),
          _p(count, torch.int32), num, _p(weights, torch.float64), S, _p(smoothed, torch.float64), _p(avg, torch.float64), _stream())
    return smoothed, avg


def instances_associate(det, valid, init, cams, center, ref_resolution, gate, max_misses, F, r, prev, live, ids, misses, next_id,
                        park, ring, count):
    """The multi-instance tracker's association for S sequences x M slots (g6d_instances_associate), rows instance-major
    (row m*S + s): det float32 [M*S,4], valid int32 [M*S], init float64 [M*S,12] (the detections' initial poses), cams
    float64 [S,20], center (3 floats).  The slot state prev float64 [M*S,12], live int32, ids int64, misses int32 [M*S],
    next_id int64 [1], park float64 [M*S,12], ring float32 [M*S,num,8,2] and count int32 [M*S] is updated in place.
    Returns (work float64 [M*2S,12], flags0 uint8 [M*2S], lists int32 [max(F,r)*M*S], det_slot int32 [M*S], spawned int32
    [M*S], dropped int64 [M*S])."""
    n, S = live.shape[0], cams.shape[0]
    M, num, dev = n // S, ring.shape[1], live.device
    if (n != M * S or det.shape != (n, 4) or valid.shape != (n,) or init.shape != (n, 12) or prev.shape != (n, 12)
            or park.shape != (n, 12) or ids.shape != (n,) or misses.shape != (n,) or next_id.shape != (1,)
            or ring.shape != (n, num, 8, 2) or count.shape != (n,)):
        raise ValueError(f'instances_associate: inconsistent shapes for {n} rows over {S} sequences')
    work = torch.empty(2 * n, 12, device=dev, dtype=torch.float64)
    flags0 = torch.empty(2 * n, device=dev, dtype=torch.uint8)
    lists = torch.empty(max(F, r) * n, device=dev, dtype=torch.int32)
    det_slot, spawned = torch.empty(n, device=dev, dtype=torch.int32), torch.empty(n, device=dev, dtype=torch.int32)
    dropped = torch.empty(n, device=dev, dtype=torch.int64)
    cx, cy, cz = (float(c) for c in center)
    _call('g6d_instances_associate', S, M, int(F), int(r), _p(det), _p(valid, torch.int32), _p(init, torch.float64),
          _p(cams, torch.float64), cx, cy, cz, float(ref_resolution), float(gate), int(max_misses), _p(prev, torch.float64),
          _p(live, torch.int32), _p(ids, torch.int64), _p(misses, torch.int32), _p(next_id, torch.int64), _p(park, torch.float64),
          _p(ring), _p(count, torch.int32), num, _p(work, torch.float64), _p(flags0, torch.uint8), _p(lists, torch.int32),
          _p(det_slot, torch.int32), _p(spawned, torch.int32), _p(dropped, torch.int64), _stream())
    return work, flags0, lists, det_slot, spawned, dropped


def instances_associate_objects(det, valid, init, cams, centers, ref_resolution, gate, max_misses, F, r, prev, live, ids, misses,
                                next_id, park, ring, count):
    """instances_associate for the K objects of an object set with M slots each (g6d_instances_associate_objects): slot
    group g = m*K + o is instance slot m of object o, and row g*S + s is that slot on sequence s.  det float32 [M*K*S,4],
    valid int32 [M*K*S], init float64 [M*K*S,12], cams float64 [S,20], centers float64 [K,3] (device); the slot state
    (prev, live, ids, misses, park, ring, count over M*K*S rows, next_id [1]) is updated in place.  Returns (work float64
    [M*K*2S,12], flags0 uint8 [M*K*2S], lists int32 [max(F,r)*M*K*S], det_slot int32, spawned int32, dropped int64
    [M*K*S])."""
    n, S, K = live.shape[0], cams.shape[0], centers.shape[0]
    M, num, dev = n // max(K * S, 1), ring.shape[1], live.device
    if (K < 1 or centers.shape != (K, 3) or n != M * K * S or det.shape != (n, 4) or valid.shape != (n,) or init.shape != (n, 12)
            or prev.shape != (n, 12) or park.shape != (n, 12) or ids.shape != (n,) or misses.shape != (n,) or next_id.shape != (1,)
            or ring.shape != (n, num, 8, 2) or count.shape != (n,)):
        raise ValueError(f'instances_associate_objects: inconsistent shapes for {n} rows over {K} objects and {S} sequences')
    work = torch.empty(2 * n, 12, device=dev, dtype=torch.float64)
    flags0 = torch.empty(2 * n, device=dev, dtype=torch.uint8)
    lists = torch.empty(max(F, r) * n, device=dev, dtype=torch.int32)
    det_slot, spawned = torch.empty(n, device=dev, dtype=torch.int32), torch.empty(n, device=dev, dtype=torch.int32)
    dropped = torch.empty(n, device=dev, dtype=torch.int64)
    _call('g6d_instances_associate_objects', S, K, M, int(F), int(r), _p(det), _p(valid, torch.int32), _p(init, torch.float64),
          _p(cams, torch.float64), _p(centers, torch.float64), float(ref_resolution), float(gate), int(max_misses),
          _p(prev, torch.float64), _p(live, torch.int32), _p(ids, torch.int64), _p(misses, torch.int32), _p(next_id, torch.int64),
          _p(park, torch.float64), _p(ring), _p(count, torch.int32), num, _p(work, torch.float64), _p(flags0, torch.uint8),
          _p(lists, torch.int32), _p(det_slot, torch.int32), _p(spawned, torch.int32), _p(dropped, torch.int64), _stream())
    return work, flags0, lists, det_slot, spawned, dropped


def instances_associate_sequences(det_index, det, valid, init, cams, centers, ref_resolution, gate, max_misses, F, r, prev, live, ids,
                                  misses, next_id, park, ring, count):
    """instances_associate_objects for a step in which only some sequences re-detect (g6d_instances_associate_sequences):
    det_index int32 [S] (device) gives each sequence its row j in a detection batch of D rows per slot group, -1 when it
    does not detect; det float32 [M*K*D,4], valid int32 [M*K*D], init float64 [M*K*D,12] (row g*D + j).  Detecting pairs
    are associated as instances_associate_objects does; the others only set up their refinement, as a refine-only step.
    Outside graph capture det_index is read back and checked (distinct rows in [0, D) or -1); inside a capture the caller
    has checked the values it uploads.  Returns (work float64 [M*K*2S,12], flags0 uint8 [M*K*2S], lists int32 [r*M*K*S +
    max(F-r,0)*M*K*D], det_slot int32, spawned int32, dropped int64 [M*K*S])."""
    from .instance_track import check_det_index, list_length
    n, S, K = live.shape[0], cams.shape[0], centers.shape[0]
    M, num, dev = n // max(K * S, 1), ring.shape[1], live.device
    D = det.shape[0] // max(M * K, 1)
    if (K < 1 or centers.shape != (K, 3) or n != M * K * S or det_index.shape != (S,) or det.shape != (M * K * D, 4)
            or valid.shape != (M * K * D,) or init.shape != (M * K * D, 12) or prev.shape != (n, 12) or park.shape != (n, 12)
            or ids.shape != (n,) or misses.shape != (n,) or next_id.shape != (1,) or ring.shape != (n, num, 8, 2)
            or count.shape != (n,)):
        raise ValueError(f'instances_associate_sequences: inconsistent shapes for {n} rows over {K} objects and {S} sequences')
    if not torch.cuda.is_current_stream_capturing():
        check_det_index(det_index.cpu().numpy(), S, D)
    work = torch.empty(2 * n, 12, device=dev, dtype=torch.float64)
    flags0 = torch.empty(2 * n, device=dev, dtype=torch.uint8)
    lists = torch.empty(list_length(M * K, S, D, int(F), int(r)), device=dev, dtype=torch.int32)
    det_slot, spawned = torch.empty(n, device=dev, dtype=torch.int32), torch.empty(n, device=dev, dtype=torch.int32)
    dropped = torch.empty(n, device=dev, dtype=torch.int64)
    _call('g6d_instances_associate_sequences', S, K, M, int(F), int(r), D, _p(det_index, torch.int32), _p(det), _p(valid, torch.int32),
          _p(init, torch.float64), _p(cams, torch.float64), _p(centers, torch.float64), float(ref_resolution), float(gate),
          int(max_misses), _p(prev, torch.float64), _p(live, torch.int32), _p(ids, torch.int64), _p(misses, torch.int32),
          _p(next_id, torch.int64), _p(park, torch.float64), _p(ring), _p(count, torch.int32), num, _p(work, torch.float64),
          _p(flags0, torch.uint8), _p(lists, torch.int32), _p(det_slot, torch.int32), _p(spawned, torch.int32),
          _p(dropped, torch.int64), _stream())
    return work, flags0, lists, det_slot, spawned, dropped


def instances_verify_update(lost, verified, max_misses, live, ids, misses):
    """A verifying instance-tracking step's slot update (g6d_instances_verify_update): lost int32 [n] (verify_judge),
    verified int32 [n] (0: a row that re-detected this step or pads the batch).  live int32, ids int64 and misses int32 [n]
    are updated in place.  Returns dropped int64 [n] (-1: none), the association's layout."""
    n = live.shape[0]
    if lost.shape != (n,) or verified.shape != (n,) or ids.shape != (n,) or misses.shape != (n,):
        raise ValueError(f'instances_verify_update: inconsistent shapes for {n} rows')
    dropped = torch.empty(n, device=live.device, dtype=torch.int64)
    _call('g6d_instances_verify_update', n, _p(lost, torch.int32), _p(verified, torch.int32), int(max_misses), _p(live, torch.int32),
          _p(ids, torch.int64), _p(misses, torch.int32), _p(dropped, torch.int64), _stream())
    return dropped


def imagenet_norm(x, out_c=4):
    out = torch.empty(*x.shape[:-1], out_c, device=x.device, dtype=torch.float32)
    _call('g6d_imagenet_norm', _p(x), _p(out), x.numel() // x.shape[-1], x.shape[-1], out_c, _stream())
    return out


def nchw_to_nhwc(x, out_c=None):
    N, Cc, H, W = x.shape
    out_c = out_c or Cc
    out = torch.empty(N, H, W, out_c, device=x.device, dtype=torch.float32)
    _call('g6d_nchw_to_nhwc', _p(x), _p(out), N, Cc, H, W, out_c, _stream())
    return out


def nhwc_to_nchw(x, channels=None):
    N, H, W, cs = x.shape
    Cc = channels or cs
    out = torch.empty(N, Cc, H, W, device=x.device, dtype=torch.float32)
    _call('g6d_nhwc_to_nchw', _p(x), _p(out), N, Cc, H, W, cs, _stream())
    return out


def resize_bilinear(x, Ho, Wo, out=None, out_coff=0):
    N, Hi, Wi, Cc = x.shape
    if out is None:
        out = torch.empty(N, Ho, Wo, Cc, device=x.device, dtype=torch.float32)
    _call('g6d_resize_bilinear', _p(x), _p(out), N, Hi, Wi, Ho, Wo, Cc, out.shape[-1], out_coff, _stream())
    return out


def resize_nearest(x, Ho, Wo):
    N, Hi, Wi, Cc = x.shape
    out = torch.empty(N, Ho, Wo, Cc, device=x.device, dtype=torch.float32)
    _call('g6d_resize_nearest', _p(x), _p(out), N, Hi, Wi, Ho, Wo, Cc, _stream())
    return out


def maxpool2x2(x):
    N, H, W, Cc = x.shape
    out = torch.empty(N, H // 2, W // 2, Cc, device=x.device, dtype=torch.float32)
    _call('g6d_maxpool2x2', _p(x), _p(out), N, H, W, Cc, _stream())
    return out


def l2norm_channels(x, eps=1e-12):
    out = torch.empty_like(x)
    _call('g6d_l2norm_channels', _p(x), _p(out), x.numel() // x.shape[-1], x.shape[-1], eps, _stream())
    return out


def instnorm_stats(x, rows_per_group, channels=None, coff=0, eps=1e-5):
    """x [..., cstride]; statistics over groups of `rows_per_group` consecutive rows.
    Returns (scale, shift), each [groups, C]: InstanceNorm(x) == x*scale + shift."""
    cstride = x.shape[-1]
    Cc = channels or cstride
    rows = x.numel() // cstride
    groups = rows // rows_per_group
    scale = torch.empty(groups, Cc, device=x.device, dtype=torch.float32)
    shift = torch.empty_like(scale)
    ws = torch.empty(groups * Cc * 2, device=x.device, dtype=torch.float64)
    _call('g6d_instnorm_stats', _p(x), rows, Cc, cstride, coff, rows_per_group, eps, _p(scale), _p(shift),
          _p(ws, torch.float64), _stream())
    return scale, shift


def instnorm_partial(x, rows_per_group, channels=None, coff=0):
    """Per (group, channel) (sum, sum of squares) as float64 [groups, C, 2] -- all-reducible across GPUs."""
    cstride = x.shape[-1]
    Cc = channels or cstride
    rows = x.numel() // cstride
    groups = rows // rows_per_group
    ws = torch.empty(groups, Cc, 2, device=x.device, dtype=torch.float64)
    _call('g6d_instnorm_partial', _p(x), rows, Cc, cstride, coff, rows_per_group, _p(ws, torch.float64), _stream())
    return ws


def instnorm_finalize(ws, count, eps=1e-5):
    """ws [groups, C, 2] (after any cross-rank reduction), count = rows per group over all ranks."""
    groups, Cc, _ = ws.shape
    scale = torch.empty(groups, Cc, device=ws.device, dtype=torch.float32)
    shift = torch.empty_like(scale)
    _call('g6d_instnorm_finalize', _p(ws, torch.float64), groups, Cc, count, eps, _p(scale), _p(shift), _stream())
    return scale, shift


def affine_act(x, scale, shift, rows_per_group, act=ACT_NONE, channels=None, in_coff=0, out=None, out_coff=0):
    ics = x.shape[-1]
    Cc = channels or ics
    rows = x.numel() // ics
    if out is None:
        out = torch.empty(*x.shape[:-1], Cc, device=x.device, dtype=torch.float32)
    _call('g6d_affine_act', _p(x), _p(out), rows, Cc, rows_per_group, _p(scale), _p(shift), act, ics, in_coff,
          out.shape[-1], out_coff, _stream())
    return out


def avgpool_affine(x, spatial, scale=None, shift=None, rows_per_group=1, act=ACT_NONE):
    """x [n_out*spatial, C] -> [n_out, C]: mean over `spatial` rows of act(x*scale+shift)."""
    Cc = x.shape[-1]
    n_out = x.numel() // Cc // spatial
    out = torch.empty(n_out, Cc, device=x.device, dtype=torch.float32)
    _call('g6d_avgpool_affine', _p(x), _p(out), n_out, spatial, Cc, rows_per_group, _p(scale), _p(shift), act, _stream())
    return out


def add(a, b):
    out = torch.empty_like(a)
    _call('g6d_add', _p(a), _p(b), _p(out), a.numel(), _stream())
    return out


# ------------------------------------------------------------------------------- convolution
@dataclass
class PackedConv:
    """Convolution weights in the library's [K, ldw] layout (+ bias), see g6d_pack_conv_weight."""
    w: Optional[torch.Tensor]   # FFMA layout (None for tensor-core-only operands)
    bias: Optional[torch.Tensor]
    cin: int          # padded input channels the packed weight expects
    cout: int
    k: tuple          # (kd, kh, kw)
    stride: int = 1
    pad: tuple = (0, 0, 0)
    w_hi: Optional[torch.Tensor] = None   # tensor-core path: [rows, K] hi / lo operand split (K-major)
    w_lo: Optional[torch.Tensor] = None
    kind: int = _lib.TC_TF32              # container of w_hi / w_lo: TC_TF32 (fp32 arrays) or TC_F16 (half arrays)
    rows: Optional[tuple] = None          # (k, rfn) of a row-decomposed detector correlation (see g6d_det_corr_rowsum)
    max_chain_k: int = 0                  # > 0: bound on the K-elements per tensor-core accumulate chain (same-sign operands)


def conv_path():
    """'tc' (wgmma split-operand kernels, default) or 'ffma' (fp32 CUDA-core fallback for A/B checks): env G6D_CONV_PATH."""
    return os.environ.get('G6D_CONV_PATH', 'tc')


def conv_kind():
    """Operand kind of the tensor-core path, env G6D_CONV_KIND: 'f16' (default; fp16 hi + 2^11-scaled fp16
    lo halves, kind::f16 MMAs: twice the K per instruction and per byte) or 'tf32' (tf32 halves: any fp32 range)."""
    return _lib.TC_TF32 if os.environ.get('G6D_CONV_KIND', 'f16') == 'tf32' else _lib.TC_F16


def tc_kind_for(cin_pad):
    """The kind a layer with `cin_pad` input channels is packed for (None: not tensor-core eligible)."""
    if cin_pad % 64 == 0 and conv_kind() == _lib.TC_F16:
        return _lib.TC_F16
    return _lib.TC_TF32 if cin_pad % 32 == 0 else None


def _tc_dtype(kind):
    return torch.float16 if kind == _lib.TC_F16 else torch.float32


def pack_conv(weight, bias=None, stride=1, pad=None, cin_pad=None, cout_scale=None, bias_override=None):
    """weight: reference layout [Cout, Cin, *k] (1-3 spatial dims) on the GPU."""
    cout, cin = weight.shape[:2]
    ks = tuple(weight.shape[2:])
    k3 = (1,) * (3 - len(ks)) + ks
    if pad is None:
        pad = tuple(kk // 2 for kk in k3)
    elif isinstance(pad, int):
        pad = tuple(pad if kk > 1 else 0 for kk in k3)
    else:
        pad = (0,) * (3 - len(pad)) + tuple(pad)
    cin_pad = cin_pad or ((cin + 3) // 4 * 4)
    taps = k3[0] * k3[1] * k3[2]
    ldw = (cout + 3) // 4 * 4
    w = weight.detach().to(torch.float32).contiguous()
    out = torch.empty(taps * cin_pad, ldw, device=w.device, dtype=torch.float32)
    _call('g6d_pack_conv_weight', _p(w), _p(out), cout, cin, cin_pad, taps,
          _p(cout_scale.contiguous()) if cout_scale is not None else None, _stream())
    b = bias_override if bias_override is not None else bias
    b = b.detach().to(torch.float32).contiguous() if b is not None else None
    pc = PackedConv(out, b, cin_pad, cout, k3, stride, pad)
    kind = tc_kind_for(cin_pad)
    if kind is not None and cout >= 16:
        rows = (cout + 7) // 8 * 8
        pc.kind = kind
        pc.w_hi = torch.empty(rows, taps * cin_pad, device=w.device, dtype=_tc_dtype(kind))
        pc.w_lo = torch.empty_like(pc.w_hi)
        _call('g6d_pack_conv_weight_tc', _p(w), _p(pc.w_hi, pc.w_hi.dtype), _p(pc.w_lo, pc.w_lo.dtype), cout, cin, cin_pad,
              taps, rows, _p(cout_scale.contiguous()) if cout_scale is not None else None, kind, _stream())
    return pc


def split_operand(x, kind=None):
    """fp32 [rows, K] -> (hi, lo, kind): the K-major B operand of the tensor-core path (detector
    reference features used as correlation kernels)."""
    kind = tc_kind_for(x.shape[-1]) if kind is None else kind
    hi = torch.empty(x.shape, device=x.device, dtype=_tc_dtype(kind))
    lo = torch.empty_like(hi)
    _call('g6d_split_operand', _p(x), _p(hi, hi.dtype), _p(lo, lo.dtype), x.numel(), kind, _stream())
    return hi, lo, kind


def transpose_to_packed(x2d):
    """[rows, K] -> packed [K, ldw(rows)] weights (detector reference features as kernels)."""
    rows, cols = x2d.shape
    out = torch.empty(cols, (rows + 3) // 4 * 4, device=x2d.device, dtype=torch.float32)
    _call('g6d_transpose2d', _p(x2d), _p(out), rows, cols, _stream())
    return out


def conv(x, pc, prologue=PRO_NONE, pro_scale=None, pro_shift=None, group_rows=1, act=ACT_NONE,
         in_coff=0, out=None, out_coff=0, stats_rows=None, prenorm=False, reuse_im2col=False, fold_splits=False,
         plan_rows=0):
    """x [B, D, H, W, cs] or [B, H, W, cs]; returns [B, Do, Ho, Wo, Cout] (or 4-D for 4-D input).
    stats_rows: also return the InstanceNorm moments of the OUTPUT, (y, ws) with ws float64
    [groups, Cout, 2] = per group of `stats_rows` consecutive output rows (sum y, sum y^2) -- fused into the
    convolution's epilogue on the tensor-core path (no extra pass over y), else by g6d_instnorm_partial;
    pass ws to instnorm_finalize (after any cross-GPU all-reduce).
    prenorm: G6D_TC_PRENORM -- a prologue layer the persistent kernel would gather takes its A operand by TMA
    im2col from a prologue-applied split copy of x instead (same result bit for bit; no-op elsewhere).
    reuse_im2col: G6D_TC_REUSE_IM2COL -- a layer the A-reuse kernel would take (and 3-D layers on the persistent
    kernel) get the split input on the persistent kernel, in the A-reuse kernel's K order (same result bit for bit).
    fold_splits: G6D_TC_FOLD_SPLITS -- a split-input layer whose tiles keep the GPU about as busy without the K splits'
    parallelism sums its splits inside the convolution instead of through fp32 partials and a reduce pass (same result
    bit for bit, smaller workspace).
    plan_rows: choose the K splits as for a call of plan_rows output rows (0: this call's own).  A call over Q groups of
    plan_rows rows (Q queries against one reference stack) then gives each group the bits a call of that group alone gives."""
    four = x.dim() == 4
    if four:
        B, H, W, cs = x.shape
        D = 1
    else:
        B, D, H, W, cs = x.shape
    kd, kh, kw = pc.k
    pd, ph, pw = pc.pad
    s = pc.stride
    Do, Ho, Wo = (D + 2 * pd - kd) // s + 1, (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
    if out is None:
        shape = (B, Ho, Wo, pc.cout) if four else (B, Do, Ho, Wo, pc.cout)
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    d = _lib.ConvDesc(B=B, D=D, H=H, W=W, Cin=pc.cin, in_cstride=cs, in_coff=in_coff, Cout=pc.cout, kd=kd, kh=kh,
                      kw=kw, stride=s, pd=pd, ph=ph, pw=pw, Do=Do, Ho=Ho, Wo=Wo, out_cstride=out.shape[-1],
                      out_coff=out_coff, prologue=prologue, group_rows=group_rows, act=act, max_chain_k=pc.max_chain_k,
                      plan_rows=plan_rows)
    work = 2.0 * B * Do * Ho * Wo * pc.cout * kd * kh * kw * pc.cin
    M = B * Do * Ho * Wo
    stats = None
    if pc.w_hi is not None and conv_path() == 'tc' and _lib.lib().g6d_conv_tc_supported(C.byref(d), pc.kind):
        flags = ((_lib.TC_PRENORM if prenorm else 0) | (_lib.TC_REUSE_IM2COL if reuse_im2col else 0)
                 | (_lib.TC_FOLD_SPLITS if fold_splits else 0))
        nbytes = _lib.lib().g6d_conv_tc_workspace_bytes_ex(C.byref(d), pc.kind, flags)
        if nbytes < 0:
            _lib.check(-1, 'g6d_conv_tc_workspace_bytes_ex')
        ws = torch.empty(nbytes // 4, device=x.device, dtype=torch.float32) if nbytes > 0 else None
        fuse = stats_rows is not None and _lib.lib().g6d_conv_tc_stats_supported(C.byref(d), pc.kind, stats_rows)
        if fuse:
            stats = torch.empty(M // stats_rows, pc.cout, 2, device=x.device, dtype=torch.float64)
        def tag(d=d, kind=pc.kind, flags=flags):        # formatted by collect_profile, outside the timed launches
            plan = (C.c_int * 6)()
            _lib.check(_lib.lib().g6d_conv_tc_plan_v2(C.byref(d), kind, flags, plan, 6), 'g6d_conv_tc_plan_v2')
            a_op = (' prenorm' if prologue != PRO_NONE else ' im2col') if plan[3] else ''
            if flags & _lib.TC_REUSE_IM2COL and plan[3]:       # '-ro': taken from the A-reuse kernel, in its K order
                plain = (C.c_int * 4)()
                _lib.check(_lib.lib().g6d_conv_tc_plan_ex(C.byref(d), kind, flags & ~_lib.TC_REUSE_IM2COL, plain),
                           'g6d_conv_tc_plan_ex')
                a_op += '-ro' if plain[0] else ''
            a_op += '-xr' if plan[5] else ''       # one A box per row of taps
            return (f'M={M} N={pc.cout} K={kd * kh * kw * pc.cin} k={kd}x{kh}x{kw} s={s} pro={prologue} '
                    f'{"reuse" if plan[0] else "persist"} BN={plan[1]} splits={plan[2]}{" fold" if plan[4] else ""}{a_op}')
        _call('g6d_conv_tc_ex', C.byref(d), _p(x), _p(pc.w_hi, pc.w_hi.dtype), _p(pc.w_lo, pc.w_lo.dtype), pc.w_hi.shape[0],
              pc.kind, _p(pc.bias), _p(pro_scale), _p(pro_shift), _p(out), _p(ws), _p(stats, torch.float64), stats_rows or 0,
              flags, _stream(), work=work, tag=tag, key='g6d_conv_tc')
    else:
        if pc.w is None:
            raise _lib.Gen6DLibraryError('this operand was packed for the tensor-core path only and the problem is not supported there')
        nbytes = _lib.lib().g6d_conv_workspace_bytes(C.byref(d))
        if nbytes < 0:
            _lib.check(-1, 'g6d_conv_workspace_bytes')
        ws = torch.empty(nbytes // 4, device=x.device, dtype=torch.float32) if nbytes > 0 else None
        _call('g6d_conv', C.byref(d), _p(x), _p(pc.w), _p(pc.bias), _p(pro_scale), _p(pro_shift), _p(out), _p(ws), _stream(),
              work=work)
    if stats_rows is None:
        return out
    if stats is None:       # not fusable here (FFMA path, groups smaller than an epilogue slice): separate pass over the output
        stats = instnorm_partial(out, rows_per_group=stats_rows, channels=pc.cout, coff=out_coff)
    return out, stats


def vgg_first_block(x, pc):
    """x [B,H,W,4] -> [B,H/2,W/2,64]: first VGG conv (BN folded) + ReLU + 2x2 max-pool in one kernel."""
    B, H, W, _ = x.shape
    out = torch.empty(B, H // 2, W // 2, 64, device=x.device, dtype=torch.float32)
    _call('g6d_vgg_first_block', _p(x), _p(pc.w), _p(pc.bias), _p(out), B, H, W, _stream())
    return out


def linear_smallm(x, w, bias, act=ACT_NONE):
    """x [M<=8, K], w [N, K] (row-major) -> [M, N]."""
    M, K = x.shape
    N = w.shape[0]
    out = torch.empty(M, N, device=x.device, dtype=torch.float32)
    _call('g6d_linear_smallm', _p(x), _p(w), _p(bias), _p(out), M, N, K, act, _stream())
    return out


# ------------------------------------------------------------------------------- detector
def det_score_fuse(maps, sizes, rfn, hs, ws, stats, clip, w1, b1, w2, b2, qn):
    """maps[s][l]: raw correlation [qn, Hl, Wl, rfn]; sizes[s][l] = (Hl, Wl). -> [qn, hs, ws, 64]."""
    m = _lib.DetMaps()
    m.n_scales, m.rfn, m.hs, m.ws = len(maps), rfn, hs, ws
    for s, lv in enumerate(maps):
        for l, t in enumerate(lv):
            m.map[s][l] = _p(t).value
            m.H[s][l], m.W[s][l] = sizes[s][l]
    for l in range(3):
        m.mu[l] = float(stats[l][0])
        m.inv_sigma[l] = 1.0 / float(stats[l][1])
    m.clip = float(clip)
    out = torch.empty(qn, hs, ws, 64, device=w1.device, dtype=torch.float32)
    _call('g6d_det_score_fuse', C.byref(m), qn, _p(w1), _p(b1), _p(w2), _p(b2), _p(out), _stream())
    return out


def det_corr_rowsum(partial, k, rfn):
    """partial [qn, H+k-1, W, k*rfn] (1 x k convolution, channel = ky*rfn + r) -> k x k correlation [qn, H, W, rfn]."""
    qn, Hp, W, _ = partial.shape
    H = Hp - (k - 1)
    out = torch.empty(qn, H, W, rfn, device=partial.device, dtype=torch.float32)
    _call('g6d_det_corr_rowsum', _p(partial), _p(out), qn, H, W, k, rfn, _stream())
    return out


def det_corr_rowsum_objects(partial, n_obj, k, rfn):
    """partial [qn, H+k-1, W, n_obj*k*rfn] (one 1 x k convolution over n_obj objects' kernels, channel = (obj*k + ky)*rfn + r)
    -> object-major k x k correlations [n_obj, qn, H, W, rfn].  k = 1: a direct correlation [qn, H, W, n_obj*rfn] regrouped."""
    qn, Hp, W, Cc = partial.shape
    if Cc != n_obj * k * rfn:
        raise ValueError(f'det_corr_rowsum_objects: {Cc} channels, expected n_obj*k*rfn = {n_obj}*{k}*{rfn}')
    H = Hp - (k - 1)
    out = torch.empty(n_obj, qn, H, W, rfn, device=partial.device, dtype=torch.float32)
    _call('g6d_det_corr_rowsum_objects', _p(partial), _p(out), n_obj, qn, H, W, k, rfn, _stream())
    return out


def det_parse(scores, scales, offsets, pool_ratio=8):
    """scores/scales [qn,hs,ws,1], offsets [qn,hs,ws,2] -> (out [qn,4] = x,y,scale,score; idx [qn] int64)."""
    qn, hs, ws, _ = scores.shape
    out = torch.empty(qn, 4, device=scores.device, dtype=torch.float32)
    idx = torch.empty(qn, device=scores.device, dtype=torch.int64)
    _call('g6d_det_parse', _p(scores), _p(scales), _p(offsets), qn, hs, ws, pool_ratio, _p(out),
          _p(idx, torch.int64), _stream())
    return out, idx


def det_parse_peaks(scores, scales, offsets, max_inst, radius=1, nms_iou=0.3, box_size=128.0, min_score=None, pool_ratio=8):
    """Up to max_inst instances per map by greedy NMS over the score-map peaks (g6d_det_parse_peaks).
    scores/scales [n,hs,ws,1], offsets [n,hs,ws,2] -> instance-major (det [max_inst,n,4] = x,y,scale,score;
    idx int64 [max_inst,n]; valid int32 [max_inst,n]; count int32 [n]).  Row 0 is det_parse's output.
    min_score None: no threshold (a raw score-head value: its meaning depends on the checkpoint)."""
    n, hs, ws, _ = scores.shape
    dev = scores.device
    det = torch.empty(max_inst, n, 4, device=dev, dtype=torch.float32)
    idx = torch.empty(max_inst, n, device=dev, dtype=torch.int64)
    valid = torch.empty(max_inst, n, device=dev, dtype=torch.int32)
    count = torch.empty(n, device=dev, dtype=torch.int32)
    _call('g6d_det_parse_peaks', _p(scores), _p(scales), _p(offsets), n, hs, ws, pool_ratio, max_inst, radius, float(nms_iou),
          float(box_size), float('-inf') if min_score is None else float(min_score), _p(det), _p(idx, torch.int64),
          _p(valid, torch.int32), _p(count, torch.int32), _stream())
    return det, idx, valid, count


def det_from_boxes(boxes, counts, max_inst, inv_box_size):
    """Detection records from caller boxes (g6d_det_from_boxes): boxes float32 [n_maps,N,5] (x0, y0, x1, y1, score),
    counts int32 [n_maps] -> instance-major (det [max_inst,n_maps,4] = x,y,scale,score; valid int32 [max_inst,n_maps];
    count int32 [n_maps]) in det_parse_peaks' layout."""
    n, N, _ = boxes.shape
    dev = boxes.device
    det = torch.empty(max_inst, n, 4, device=dev, dtype=torch.float32)
    valid = torch.empty(max_inst, n, device=dev, dtype=torch.int32)
    count = torch.empty(n, device=dev, dtype=torch.int32)
    _call('g6d_det_from_boxes', _p(boxes), _p(counts, torch.int32), n, N, max_inst, float(inv_box_size), _p(det),
          _p(valid, torch.int32), _p(count, torch.int32), _stream())
    return det, valid, count


# ------------------------------------------------------------------------------- selector
def sel_ref_sums(ref):
    """ref [S, P, C] -> (sum, sum of squares) over S, float64 [P, C]."""
    S, Pn, Cc = ref.shape
    s1 = torch.empty(Pn, Cc, device=ref.device, dtype=torch.float64)
    s2 = torch.empty_like(s1)
    _call('g6d_sel_ref_sums', _p(ref), S, Pn, Cc, _p(s1, torch.float64), _p(s2, torch.float64), _stream())
    return s1, s2


def sel_corr_prologue(q, s1, s2, S, eps=1e-5):
    Pn, Cc = q.shape
    scale = torch.empty(Pn, Cc, device=q.device, dtype=torch.float32)
    shift = torch.empty(Cc, device=q.device, dtype=torch.float32)
    _call('g6d_sel_corr_prologue', _p(q), _p(s1, torch.float64), _p(s2, torch.float64), S, Pn, Cc, eps, _p(scale),
          _p(shift), _stream())
    return scale, shift


def sel_corr_score(ref, q, out=None):
    S, Pn, Cc = ref.shape
    if out is None:
        out = torch.empty(S, device=ref.device, dtype=torch.float32)
    _call('g6d_sel_corr_score', _p(ref), _p(q), S, Pn, Cc, _p(out), _stream(),
          work=4.0 * (S * Pn * Cc + Pn * Cc + S))
    return out


def sel_corr_score3(refs, qs, counters=None, out=None):
    """refs: 3 x [S, P_l, C]; qs: 3 x [P_l, C] -> score [3, S] in one streaming pass (into `out` when given).
    counters: int32 [3*S], zero (the kernel leaves it zero): one launch; None: dots + finish kernels."""
    S, Cc = refs[0].shape[0], refs[0].shape[2]
    Ps = [r.shape[1] for r in refs]
    if out is None:
        out = torch.empty(3, S, device=refs[0].device, dtype=torch.float32)
    ws = torch.empty(_lib.lib().g6d_sel_corr_score3_workspace_bytes(S, *Ps) // 4, device=refs[0].device, dtype=torch.float32)
    _call('g6d_sel_corr_score3', _p(refs[0]), _p(refs[1]), _p(refs[2]), _p(qs[0]), _p(qs[1]), _p(qs[2]), S, Ps[0], Ps[1],
          Ps[2], Cc, _p(out), _p(ws), _p(counters, torch.int32), _stream(), work=4.0 * (S * sum(Ps) * Cc + sum(Ps) * Cc + 3 * S))
    return out


def sel_vp_norm(score, feats, coff, eps=1e-5):
    Ln, n = score.shape
    _call('g6d_sel_vp_norm', _p(score), Ln, n, eps, _p(feats), feats.shape[-1], coff, _stream())


def sel_max_angle_add(x, embed, out=None):
    rfn, an, Cc = x.shape
    if out is None:
        out = torch.empty(rfn, Cc, device=x.device, dtype=torch.float32)
    _call('g6d_sel_max_angle_add', _p(x), _p(embed), _p(out), rfn, an, Cc, _stream())
    return out


def attention(q, k, v, heads, head_major=False, out=None):
    """q, k, v [n, C] -> [n, C] (into `out` when given).  head_major=False: the reference's channel order
    c = d*heads + head; True: c = head*D + d (the tiled kernel; producers / consumer permuted at pack time)."""
    n, Cc = q.shape
    if out is None:
        out = torch.empty_like(q)
    _call('g6d_attention_headmajor' if head_major else 'g6d_attention', _p(q), _p(k), _p(v), _p(out), n, Cc, heads, _stream())
    return out


def layernorm(x, gamma, beta, eps=1e-5):
    rows, Cc = x.shape
    out = torch.empty_like(x)
    _call('g6d_layernorm', _p(x), _p(gamma), _p(beta), _p(out), rows, Cc, eps, _stream())
    return out


def sel_parse(logits, angles):
    qn, rfn = logits.shape
    idx = torch.empty(qn, device=logits.device, dtype=torch.int64)
    out = torch.empty(qn, 2, device=logits.device, dtype=torch.float32)
    _call('g6d_sel_parse', _p(logits), _p(angles), qn, rfn, _p(idx, torch.int64), _p(out), _stream())
    return idx, out


# ------------------------------------------------------------------------------- refiner
def ref_volume_fill(ref_feats, que_feats, ref_Ks, ref_poses, que_Ks, que_poses, sn, img_h, img_w):
    Q, R, fh, fw, Cc = ref_feats.shape
    mean_in = torch.empty(Q, sn, sn, sn, 2 * Cc, device=ref_feats.device, dtype=torch.float32)
    stdv = torch.empty(Q, sn, sn, sn, Cc, device=ref_feats.device, dtype=torch.float32)
    _call('g6d_ref_volume_fill', _p(ref_feats), _p(que_feats), _p(ref_Ks), _p(ref_poses), _p(que_Ks), _p(que_poses),
          Q, R, fh, fw, Cc, sn, img_h, img_w, _p(mean_in), _p(stdv), _stream(),
          work=4.0 * Q * ((R + 1) * fh * fw * Cc + 3 * Cc * sn ** 3))
    return mean_in, stdv


def ref_pose_heads(x, w, b):
    M, K = x.shape
    out = torch.empty(M, 7, device=x.device, dtype=torch.float32)
    _call('g6d_ref_pose_heads', _p(x), _p(w), _p(b), _p(out), M, K, _stream())
    return out
