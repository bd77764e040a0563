"""Numpy restatement of g6d_det_from_boxes (include/gen6d_b200.h): caller boxes -> detection records in
g6d_det_parse_peaks' instance-major layout."""
import numpy as np


def records(boxes, counts, max_inst, inv_box_size):
    """boxes float32 [n_maps, N, 5] (x0, y0, x1, y1, score), counts [n_maps] -> (det float32 [max_inst, n_maps, 4], valid
    int32 [max_inst, n_maps], count int32 [n_maps])."""
    boxes = np.asarray(boxes, np.float32)
    n, N, _ = boxes.shape
    det = np.zeros((max_inst, n, 4), np.float32)
    valid, count = np.zeros((max_inst, n), np.int32), np.zeros(n, np.int32)
    half, inv = np.float32(0.5), np.float32(inv_box_size)
    for j in range(n):
        b = boxes[j, :min(max(int(counts[j]), 0), N)]
        with np.errstate(invalid='ignore', over='ignore'):
            usable = np.isfinite(b).all(1) & (b[:, 2] > b[:, 0]) & (b[:, 3] > b[:, 1])
            s, i = b[:, 4], np.arange(len(b))
            # rank of a usable box: the usable boxes before it, by score descending, ties to the lower index
            before = usable[None, :] & ((s[None, :] > s[:, None]) | ((s[None, :] == s[:, None]) & (i[None, :] < i[:, None])))
            rank = before.sum(1)
            w, h = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
            rec = np.stack([(b[:, 0] + b[:, 2]) * half, (b[:, 1] + b[:, 3]) * half, np.where(w > h, w, h) * inv, s], 1)
        row0 = np.array([0, 0, 1, -np.inf], np.float32)
        k = 0
        for bi in np.flatnonzero(usable):
            if rank[bi] < max_inst:
                det[rank[bi], j], valid[rank[bi], j] = rec[bi], 1
                k += 1
                if rank[bi] == 0:
                    row0 = rec[bi]
        det[k:, j], valid[k:, j], count[j] = row0, 0, k
    return det, valid, count


def random_table(rng, n_maps, N, frame=(480, 640)):
    """A seeded box table exercising every rule: counts 0..N, tied scores, NaN and +-inf in coordinates and scores, zero
    and negative widths and heights, boxes larger than the frame."""
    h, w = frame
    x0 = rng.uniform(-100, w + 100, (n_maps, N)).astype(np.float32)
    y0 = rng.uniform(-100, h + 100, (n_maps, N)).astype(np.float32)
    bw = rng.choice([rng.uniform(1, 300), 0.0, -5.0, 4 * w, 1e30], (n_maps, N), p=[0.7, 0.08, 0.08, 0.09, 0.05])
    bh = rng.choice([rng.uniform(1, 300), 0.0, -3.0, 4 * h], (n_maps, N), p=[0.75, 0.08, 0.08, 0.09])
    scores = rng.choice([0.0, -0.0, 0.25, 0.5, 0.9, 1.0], (n_maps, N)).astype(np.float32)
    scores += (rng.rand(n_maps, N) < 0.5) * rng.rand(n_maps, N).astype(np.float32)
    t = np.stack([x0, y0, x0 + bw.astype(np.float32), y0 + bh.astype(np.float32), scores], 2).astype(np.float32)
    bad = rng.rand(n_maps, N, 5) < 0.03
    t[bad] = rng.choice([np.nan, np.inf, -np.inf], bad.sum())
    counts = rng.randint(0, N + 1, n_maps).astype(np.int32)
    counts[0], counts[-1] = 0, N
    return t, counts
