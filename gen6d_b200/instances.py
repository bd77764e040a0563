"""Shared pieces of the multi-instance predictions (Gen6DEstimator.predict_instances, ObjectSet.predict_instances).

Instances are slots: the detector's score-map peaks (g6d_det_parse_peaks) come out instance-major, so with K objects on
qn frames row m*K*qn + o*qn + f is instance m of object o on frame f, i.e. slot s = m*K + o in the object-major layout
the g6d_glue_*_objects launches take (every slot of object o passes object o's view table).  A slot row whose instance was
not found still runs through crop, selection and refinement on a repeat of instance 0's detection, so the graph has
fixed shapes; instance_valid masks it.
"""
import numpy as np
import torch

from . import _lib


def check_args(max_instances, nms_iou, peak_radius, min_score):
    """-> the part of a graph's key these arguments set; ValueError for values g6d_det_parse_peaks rejects."""
    if not isinstance(max_instances, (int, np.integer)) or not 1 <= max_instances <= _lib.G6D_DET_MAX_INSTANCES:
        raise ValueError(f'max_instances={max_instances!r}: need an integer in [1, {_lib.G6D_DET_MAX_INSTANCES}]')
    if not isinstance(peak_radius, (int, np.integer)) or not 0 <= peak_radius <= _lib.G6D_DET_MAX_PEAK_RADIUS:
        raise ValueError(f'peak_radius={peak_radius!r}: need an integer in [0, {_lib.G6D_DET_MAX_PEAK_RADIUS}]')
    if not 0.0 <= float(nms_iou) <= 1.0:
        raise ValueError(f'nms_iou={nms_iou!r}: need a value in [0, 1]')
    if min_score is not None and np.isnan(float(min_score)):
        raise ValueError('min_score is NaN: pass None for no threshold')
    # as float32, the values the kernel compares with
    return (int(max_instances), int(peak_radius), float(np.float32(nms_iou)),
            None if min_score is None else float(np.float32(min_score)))


def pack(parts, crop):
    """Device tensors -> one uint8 buffer (every part as float64, then the crops' bytes): the call's single read."""
    packed = torch.cat([t.reshape(-1).to(torch.float64) for t in parts])
    return torch.cat([packed.view(torch.uint8), crop.reshape(-1)])


class Unpacker:
    """Reads pack()'s buffer back on the host in the order it was packed."""

    def __init__(self, host, crop_bytes):
        self.f64 = host[:len(host) - crop_bytes].view(np.float64)
        self.crops = host[len(host) - crop_bytes:]
        self.off = 0

    def take(self, n):
        self.off += n
        return self.f64[self.off - n:self.off]


def frame_major(a, M, qn):
    """[M*qn, ...] instance-major rows -> [qn, M, ...] (a contiguous copy)."""
    a = a.reshape(M, qn, *a.shape[1:])
    return np.ascontiguousarray(np.swapaxes(a, 0, 1))


def inter_of(chain, det, idx, sel_out, logits, valid, count, crops, M, qn):
    """Instance-major host arrays of one object -> (poses [qn,M,3,4], inter with predict_batch's keys led by [qn, M])."""
    fm = lambda a: frame_major(a, M, qn)
    chain = [fm(c.reshape(M * qn, 3, 4)) for c in chain]
    refined = [c.astype(np.float32) for c in chain[1:]]
    det = fm(det.reshape(M * qn, 4).astype(np.float32))
    sel_out = fm(sel_out.reshape(M * qn, 2).astype(np.float32))
    inter = {'det_position': np.ascontiguousarray(det[..., :2]), 'det_scale_r2q': np.ascontiguousarray(det[..., 2]),
             'det_score': np.ascontiguousarray(det[..., 3]), 'det_que_img': fm(crops),
             'sel_angle_r2q': np.ascontiguousarray(sel_out[..., 0]), 'sel_scores': fm(logits.reshape(M * qn, -1).astype(np.float32)),
             'sel_ref_idx': fm(idx.reshape(M * qn).astype(np.int64)), 'refine_poses': [chain[0]] + refined,
             'instance_valid': fm(valid.reshape(M * qn).astype(bool)), 'instance_count': count.astype(np.int64)}
    return (refined[-1] if refined else chain[0]), inter
