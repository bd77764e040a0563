"""Tables and call wrappers of the device-side camera algebra (csrc/glue.cu, include/gen6d_b200.h g6d_glue_*).

Between the stages of a prediction the reference's estimator does small camera computations on the host
(estimator.py:176-214).  geometry.py restates them in numpy; csrc/glue_math.cuh restates them once more as
__host__ __device__ code so that a batched prediction can stay on the GPU from the uploaded frames to the final
poses.  This module builds what those kernels read:
  * cameras(que_Ks): per-frame constants that depend on K only (K, np.linalg.inv(K), (K00 + K11) / 2, each evaluated
    by numpy in K's own dtype, handed over as float64 values);
  * selector_refs(ref_info): per selector reference view, what poses_from_similarity needs of it;
  * refiner_views(database, ref_ids, ...): the pose-independent view table of geometry.NormalizedView, the FPS
    re-spread subset with its viewing directions, and the unit-sphere normalisation.
The `host_*` functions run the library's *_host entry points on numpy arrays: same code as the kernels, no GPU --
tests/test_glue.py pins them against geometry.py.
"""
import ctypes as C

import numpy as np

from . import _lib
from . import geometry as G

JOB = G.WARP_JOB


def cameras(que_Ks):
    """[qn,3,3] intrinsics (any float dtype) -> float64 [qn,20] = g6d_glue_camera records."""
    Ks = np.asarray(que_Ks)
    out = np.zeros((len(Ks), 20), np.float64)
    out[:, :9] = Ks.reshape(len(Ks), 9)
    out[:, 9:18] = np.linalg.inv(Ks).reshape(len(Ks), 9)
    f = (Ks[:, 0, 0] + Ks[:, 1, 1]) / 2
    out[:, 18], out[:, 19] = f, f ** 2
    return out


def selector_refs(ref_info):
    """estimator.ref_info -> arrays of g6d_glue_refs (what geometry.poses_from_similarity reads per reference view)."""
    poses, Ks = np.asarray(ref_info['poses']), np.asarray(ref_info['Ks'])
    center = np.asarray(ref_info['center'], np.float64)
    return {'poses': np.ascontiguousarray(poses.reshape(len(poses), 12), np.float64),
            'cen': np.ascontiguousarray(G._project_center_batch(center, poses, Ks), np.float64),
            'f': np.ascontiguousarray((Ks[:, 0, 0] + Ks[:, 1, 1]) / 2, np.float64),
            'dist': np.asarray([np.linalg.norm(G.camera_center(p) - center) for p in poses], np.float64),
            'center': center}


def refiner_views(database, ref_ids, size=128, ref_num=6, margin=0.05):
    """The refiner's view tables (g6d_glue_views minus the image addresses) for refine_problems(ref_even=True)."""
    view = G._normalized_view(database)
    ids = list(ref_ids)
    tab = view.view_table(ids, size, margin, prefill=ids)
    center = view.object_center()
    ids_e, _, dirs = view.even_subset(ids, min(128, len(ids)), center)
    row = {i: k for k, i in enumerate(ids)}
    n = len(ids)
    return {'ids': ids, 'view': view,
            'poses': np.ascontiguousarray(tab['poses'].reshape(n, 12), np.float64),
            'R_look': np.ascontiguousarray(tab['R_look'].reshape(n, 9), np.float64),
            'RlookR': np.ascontiguousarray(tab['RlookR'].reshape(n, 9), np.float64),
            'f': np.ascontiguousarray(tab['f'], np.float64),
            'Kinv': np.ascontiguousarray(tab['Kinv'].reshape(n, 9), np.float64),
            'even_idx': np.asarray([row[i] for i in ids_e], np.int32),
            'even_dirs': np.ascontiguousarray(dirs, np.float32),
            'norm_scale': float(view.scale), 'norm_offset': np.asarray(view.offset, np.float32),
            'size_scale': np.float32(size * (1 - margin) / view.object_diameter()), 'size': size, 'ref_num': ref_num}


# ------------------------------------------------------------------------------------------ struct packing
def _ptr(a):
    return a.ctypes.data if isinstance(a, np.ndarray) else int(a)


def refs_struct(arr):
    """arr: dict of numpy arrays (host entry points) or of device addresses."""
    s = _lib.GlueRefs()
    s.poses, s.cen, s.f, s.dist = _ptr(arr['poses']), _ptr(arr['cen']), _ptr(arr['f']), _ptr(arr['dist'])
    s.center[:] = [float(v) for v in arr['center']]
    return s


def views_struct(arr, tables, src=0, rows=0, cols=0):
    """arr: addresses (numpy arrays or device pointers) of the per-view arrays; tables: the refiner_views() dict."""
    s = _lib.GlueViews()
    for k in ('poses', 'R_look', 'RlookR', 'f', 'Kinv', 'even_idx', 'even_dirs'):
        setattr(s, k, _ptr(arr[k]))
    s.src, s.rows, s.cols = _ptr(src), _ptr(rows), _ptr(cols)
    s.n_views, s.n_even, s.ref_num, s.size = len(tables['ids']), len(tables['even_idx']), tables['ref_num'], tables['size']
    s.norm_scale = tables['norm_scale']
    s.norm_offset[:] = [float(v) for v in tables['norm_offset']]
    s.size_scale = float(tables['size_scale'])
    return s


# ------------------------------------------------------------------------------------------ host entry points (tests)
def host_detection_jobs(det_out, rows, cols, size, frame_ptr=0):
    det = np.ascontiguousarray(det_out, np.float32)
    jobs = np.zeros(len(det), JOB)
    _lib.check(_lib.lib().g6d_glue_detection_jobs_host(det.ctypes.data, frame_ptr, rows, cols, len(det), size, jobs.ctypes.data),
               'g6d_glue_detection_jobs_host')
    return jobs


def host_initial_poses(det_out, sel_idx, sel_out, refs, cams):
    det, idx = np.ascontiguousarray(det_out, np.float32), np.ascontiguousarray(sel_idx, np.int64)
    so, cams = np.ascontiguousarray(sel_out, np.float32), np.ascontiguousarray(cams, np.float64)
    poses = np.zeros((len(det), 3, 4), np.float64)
    st = refs_struct(refs)
    _lib.check(_lib.lib().g6d_glue_initial_poses_host(det.ctypes.data, idx.ctypes.data, so.ctypes.data, C.byref(st), cams.ctypes.data,
                                                      len(det), poses.ctypes.data), 'g6d_glue_initial_poses_host')
    return poses


def host_refine_problems(tables, cams, poses, poses_are_f32, rows, cols, frame_ptr=0, src=None, img_rows=None, img_cols=None):
    n, R = len(poses), tables['ref_num']
    nv = len(tables['ids'])
    src = np.zeros(nv, np.uint64) if src is None else np.ascontiguousarray(src, np.uint64)
    img_rows = np.zeros(nv, np.int32) if img_rows is None else np.ascontiguousarray(img_rows, np.int32)
    img_cols = np.zeros(nv, np.int32) if img_cols is None else np.ascontiguousarray(img_cols, np.int32)
    st = views_struct(tables, tables, src, img_rows, img_cols)
    cams, poses = np.ascontiguousarray(cams, np.float64), np.ascontiguousarray(poses, np.float64)
    out = {'jobs': np.zeros(n * (R + 1), JOB), 'que_K': np.zeros((n, 3, 3), np.float32), 'que_pose': np.zeros((n, 3, 4), np.float32),
           'pose_rect': np.zeros((n, 3, 4), np.float32), 'ref_Ks': np.zeros((n, R, 3, 3), np.float32),
           'ref_poses': np.zeros((n, R, 3, 4), np.float32), 'ref_rows': np.zeros((n, R), np.int32)}
    _lib.check(_lib.lib().g6d_glue_refine_problems_host(C.byref(st), cams.ctypes.data, frame_ptr, rows, cols, poses.ctypes.data,
                                                        int(poses_are_f32), n, *[out[k].ctypes.data for k in
                                                                                 ('jobs', 'que_K', 'que_pose', 'pose_rect', 'ref_Ks',
                                                                                  'ref_poses', 'ref_rows')]),
               'g6d_glue_refine_problems_host')
    return out


def host_apply_refinements(tables, prob, net_out):
    st = views_struct(tables, tables)
    net = np.ascontiguousarray(net_out, np.float32)
    poses = np.zeros((len(net), 3, 4), np.float64)
    _lib.check(_lib.lib().g6d_glue_apply_refinements_host(C.byref(st), prob['que_pose'].ctypes.data, prob['que_K'].ctypes.data,
                                                          prob['pose_rect'].ctypes.data, net.ctypes.data, len(net), poses.ctypes.data),
               'g6d_glue_apply_refinements_host')
    return poses


def _views_array(structs):
    return (_lib.GlueViews * len(structs))(*structs)


def host_refine_problems_objects(tables_list, cams, poses, poses_are_f32, rows, cols, frame_ptr=0, sources=None):
    """g6d_glue_refine_problems_objects_host: K objects' tables, cams [qn,20], poses [K*qn,3,4] object-major (row o*qn + s
    is object o on frame s) -> the outputs of host_refine_problems, K*qn rows.  sources: per object (src, img_rows,
    img_cols) of its views, as host_refine_problems takes them (default zeros)."""
    K, qn = len(tables_list), len(cams)
    n, R = len(poses), tables_list[0]['ref_num']
    if sources is None:
        sources = [(None, None, None)] * K
    keep = []
    for t, (src, img_rows, img_cols) in zip(tables_list, sources):
        nv = len(t['ids'])
        keep.append((np.zeros(nv, np.uint64) if src is None else np.ascontiguousarray(src, np.uint64),
                     np.zeros(nv, np.int32) if img_rows is None else np.ascontiguousarray(img_rows, np.int32),
                     np.zeros(nv, np.int32) if img_cols is None else np.ascontiguousarray(img_cols, np.int32)))
    views = _views_array([views_struct(t, t, *k) for t, k in zip(tables_list, keep)])
    cams, poses = np.ascontiguousarray(cams, np.float64), np.ascontiguousarray(poses, np.float64)
    out = {'jobs': np.zeros(n * (R + 1), JOB), 'que_K': np.zeros((n, 3, 3), np.float32), 'que_pose': np.zeros((n, 3, 4), np.float32),
           'pose_rect': np.zeros((n, 3, 4), np.float32), 'ref_Ks': np.zeros((n, R, 3, 3), np.float32),
           'ref_poses': np.zeros((n, R, 3, 4), np.float32), 'ref_rows': np.zeros((n, R), np.int32)}
    _lib.check(_lib.lib().g6d_glue_refine_problems_objects_host(views, K, qn, cams.ctypes.data, frame_ptr, rows, cols, poses.ctypes.data,
                                                                int(poses_are_f32), *[out[k].ctypes.data for k in
                                                                                      ('jobs', 'que_K', 'que_pose', 'pose_rect', 'ref_Ks',
                                                                                       'ref_poses', 'ref_rows')]),
               'g6d_glue_refine_problems_objects_host')
    return out


def host_apply_refinements_objects(tables_list, prob, net_out):
    """g6d_glue_apply_refinements_objects_host: K objects' tables, the K*qn problems of host_refine_problems_objects and
    network outputs [K*qn,7] -> refined poses [K*qn,3,4]."""
    K = len(tables_list)
    views = _views_array([views_struct(t, t) for t in tables_list])
    net = np.ascontiguousarray(net_out, np.float32)
    poses = np.zeros((len(net), 3, 4), np.float64)
    _lib.check(_lib.lib().g6d_glue_apply_refinements_objects_host(views, K, len(net) // K, prob['que_pose'].ctypes.data,
                                                                  prob['que_K'].ctypes.data, prob['pose_rect'].ctypes.data,
                                                                  net.ctypes.data, poses.ctypes.data),
               'g6d_glue_apply_refinements_objects_host')
    return poses


def host_refine_problems_rows(tables_list, cams, poses, row_idx, row_f32, rows, cols, frame_ptr=0, sources=None):
    """g6d_glue_refine_problems_rows_host: poses [K*qn,3,4] object-major as host_refine_problems_objects takes them, row_idx
    [n_sel] the listed rows, row_f32 [K*qn] each row's dtype flag -> the outputs of host_refine_problems for the n_sel
    listed rows, output row j being row row_idx[j]."""
    K, qn = len(tables_list), len(cams)
    R = tables_list[0]['ref_num']
    if sources is None:
        sources = [(None, None, None)] * K
    keep = []
    for t, (src, img_rows, img_cols) in zip(tables_list, sources):
        nv = len(t['ids'])
        keep.append((np.zeros(nv, np.uint64) if src is None else np.ascontiguousarray(src, np.uint64),
                     np.zeros(nv, np.int32) if img_rows is None else np.ascontiguousarray(img_rows, np.int32),
                     np.zeros(nv, np.int32) if img_cols is None else np.ascontiguousarray(img_cols, np.int32)))
    views = _views_array([views_struct(t, t, *k) for t, k in zip(tables_list, keep)])
    cams, poses = np.ascontiguousarray(cams, np.float64), np.ascontiguousarray(poses, np.float64)
    idx, flags = np.ascontiguousarray(row_idx, np.int32), np.ascontiguousarray(row_f32, np.uint8)
    n = len(idx)
    out = {'jobs': np.zeros(n * (R + 1), JOB), 'que_K': np.zeros((n, 3, 3), np.float32), 'que_pose': np.zeros((n, 3, 4), np.float32),
           'pose_rect': np.zeros((n, 3, 4), np.float32), 'ref_Ks': np.zeros((n, R, 3, 3), np.float32),
           'ref_poses': np.zeros((n, R, 3, 4), np.float32), 'ref_rows': np.zeros((n, R), np.int32)}
    _lib.check(_lib.lib().g6d_glue_refine_problems_rows_host(views, K, qn, cams.ctypes.data, frame_ptr, rows, cols, poses.ctypes.data,
                                                             idx.ctypes.data, n, flags.ctypes.data,
                                                             *[out[k].ctypes.data for k in ('jobs', 'que_K', 'que_pose', 'pose_rect',
                                                                                            'ref_Ks', 'ref_poses', 'ref_rows')]),
               'g6d_glue_refine_problems_rows_host')
    return out


def host_apply_refinements_rows(tables_list, prob, net_out, row_idx, poses):
    """g6d_glue_apply_refinements_rows_host: the n_sel problems of host_refine_problems_rows and network outputs [n_sel,7]
    update rows row_idx of poses (float64 [K*qn,3,4], contiguous, in place).  Returns poses."""
    K = len(tables_list)
    views = _views_array([views_struct(t, t) for t in tables_list])
    net, idx = np.ascontiguousarray(net_out, np.float32), np.ascontiguousarray(row_idx, np.int32)
    if poses.dtype != np.float64 or not poses.flags.c_contiguous or len(poses) % K:
        raise ValueError('host_apply_refinements_rows: poses must be a contiguous float64 array of K*qn rows (updated in place)')
    _lib.check(_lib.lib().g6d_glue_apply_refinements_rows_host(views, K, len(poses) // K, prob['que_pose'].ctypes.data,
                                                               prob['que_K'].ctypes.data, prob['pose_rect'].ctypes.data, net.ctypes.data,
                                                               idx.ctypes.data, len(idx), poses.ctypes.data),
               'g6d_glue_apply_refinements_rows_host')
    return poses
