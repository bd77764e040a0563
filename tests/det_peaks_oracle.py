"""Numpy restatement of g6d_det_parse_peaks (include/gen6d_b200.h): every instance of the object in a score map by greedy
non-maximum suppression over its peaks.  Written from the header's definition, not from the kernel: the order is
argsort-based, the peak test compares ranks over a padded window, and the NMS walks the sorted peaks once."""
import numpy as np

F32 = np.float32


def _fma32(a, b, c):
    """float32 fma(a, b, c): the float64 product of two float32 values is exact, and so is adding c at the magnitudes of a
    detector map (|a*b| < 2^24), so one rounding to float32 gives the fused result."""
    return F32(np.float64(a) * np.float64(b) + np.float64(c))


def exp2_f64(v):
    return F32(np.exp2(np.float64(v)))


def order(sc):
    """Flat indices of sc sorted by g6d_det_parse's order: NaN first, then descending value, ties by ascending index."""
    sc = np.asarray(sc, F32).reshape(-1)
    nan = np.isnan(sc)
    key = np.where(nan, F32(0), -sc)
    return np.lexsort((np.arange(sc.size), key, ~nan))


def peaks(sc, radius):
    """bool [hs, ws]: no other cell within Chebyshev distance `radius` (clipped window) comes before the cell."""
    hs, ws = sc.shape
    rank = np.empty(hs * ws, np.int64)
    rank[order(sc)] = np.arange(hs * ws)
    rank = rank.reshape(hs, ws)
    big = np.iinfo(np.int64).max
    pad = np.full((hs + 2 * radius, ws + 2 * radius), big, np.int64)
    pad[radius:radius + hs, radius:radius + ws] = rank
    ok = np.ones((hs, ws), bool)
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            if dy or dx:
                ok &= rank < pad[radius + dy:radius + dy + hs, radius + dx:radius + dx + ws]
    return ok


def decode(sc, scl, off, idx, pool, exp2):
    ws = sc.shape[1]
    y, x = divmod(int(idx), ws)
    ox, oy = off[y, x, 0], off[y, x, 1]
    return np.array([_fma32(F32(F32(x) + ox) + F32(0.5), F32(pool), F32(-0.5)),
                     _fma32(F32(F32(y) + oy) + F32(0.5), F32(pool), F32(-0.5)),
                     exp2(scl[y, x]), sc[y, x]], F32)


def box(d, box_size):
    side = F32(box_size) * d[2]
    half = side * F32(0.5)
    return (d[0] - half, d[1] - half, d[0] + half, d[1] + half, side * side)


def iou(a, b):
    with np.errstate(invalid='ignore', divide='ignore'):
        iw = np.fmax(np.fmin(a[2], b[2]) - np.fmax(a[0], b[0]), F32(0))
        ih = np.fmax(np.fmin(a[3], b[3]) - np.fmax(a[1], b[1]), F32(0))
        inter = iw * ih
        return F32(inter / ((a[4] + b[4]) - inter))


def det_peaks(scores, scales, offsets, pool_ratio=8, max_inst=4, radius=1, nms_iou=0.3, box_size=128.0, min_score=-np.inf,
              exp2=exp2_f64, trace=None):
    """scores/scales [n, hs, ws] (a trailing 1 is dropped), offsets [n, hs, ws, 2] ->
    (det float32 [max_inst, n, 4], idx int64 [max_inst, n], valid int32 [max_inst, n], count int32 [n]).
    exp2: float32 -> float32 scale decode (the device uses ex2.approx, the host twin libm's exp2f).
    trace: a list that receives every IoU the greedy pass compares with nms_iou (the decisions the result rests on)."""
    scores, scales = np.asarray(scores, F32), np.asarray(scales, F32)
    if scores.ndim == 4:
        scores, scales = scores[..., 0], scales[..., 0]
    offsets = np.asarray(offsets, F32)
    n = scores.shape[0]
    thr, nms_iou = F32(min_score), F32(nms_iou)
    det = np.zeros((max_inst, n, 4), F32)
    idx = np.zeros((max_inst, n), np.int64)
    valid = np.zeros((max_inst, n), np.int32)
    count = np.zeros(n, np.int32)
    for j in range(n):
        sc, scl, off = scores[j], scales[j], offsets[j]
        srt = order(sc)
        first = decode(sc, scl, off, srt[0], pool_ratio, exp2)
        keep = [(int(srt[0]), first)]
        if first[3] >= thr:
            pk = peaks(sc, radius).reshape(-1)
            for i in srt[1:]:
                if len(keep) == max_inst:
                    break
                if not pk[i] or not sc.reshape(-1)[i] >= thr:
                    continue
                d = decode(sc, scl, off, i, pool_ratio, exp2)
                b = box(d, box_size)
                ious = [iou(box(k[1], box_size), b) for k in keep]
                if trace is not None:
                    trace.extend(ious)
                if all(not v > nms_iou for v in ious):
                    keep.append((int(i), d))
            count[j] = len(keep)
        for m in range(max_inst):
            i, d = keep[m] if m < len(keep) else keep[0]
            det[m, j], idx[m, j] = d, i
            valid[m, j] = int(m < count[j])
    return det, idx, valid, count


def box_ious(scores, scales, offsets, pool_ratio=8, box_size=128.0, exp2=exp2_f64, cells=None):
    """IoU of every pair of the given cells' boxes (all cells by default) of each map: list of float32 [c, c]."""
    scores, scales = np.asarray(scores, F32), np.asarray(scales, F32)
    if scores.ndim == 4:
        scores, scales = scores[..., 0], scales[..., 0]
    out = []
    for j in range(scores.shape[0]):
        cs = range(scores[j].size) if cells is None else cells[j]
        bs = [box(decode(scores[j], scales[j], offsets[j], i, pool_ratio, exp2), box_size) for i in cs]
        out.append(np.array([[iou(a, b) for b in bs] for a in bs], F32).reshape(len(bs), len(bs)))
    return out
