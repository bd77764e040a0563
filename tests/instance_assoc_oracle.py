"""numpy restatement of g6d_instances_associate (the multi-instance tracker's re-detection step), written independently
of the kernel: the greedy matching is stated as "sort every admissible pair by (cost, slot, detection) and accept the
pairs whose slot and detection are both still free", which picks the same pairs as repeated smallest-cost extraction.
Every fp64 operation is spelled out in the kernel's order; numpy rounds each product and sum separately."""
import numpy as np


def track_points(prev, K, center):
    """prev [M,12], K [9], center [3] -> (u [M], v [M], ok [M]): the object centre projected with each pose."""
    P = prev.reshape(-1, 3, 4)
    cx, cy, cz = (np.float64(c) for c in center)
    p = [((P[:, i, 0] * cx + P[:, i, 1] * cy) + P[:, i, 2] * cz) + P[:, i, 3] for i in range(3)]
    q = [(K[j * 3] * p[0] + K[j * 3 + 1] * p[1]) + K[j * 3 + 2] * p[2] for j in range(3)]
    ok = ~(q[2] <= 0)
    with np.errstate(divide='ignore', invalid='ignore'):
        return q[0] / q[2], q[1] / q[2], ok


def associate(det, valid, init, cams, center, res, gate, max_misses, F, r, prev, live, ids, misses, next_id, park, ring, count):
    """Same arguments and results as instance_track.host_associate; the state arrays are updated in place."""
    n, S = len(live), len(cams)
    M = n // S
    work, flags0 = np.zeros((M, 2 * S, 12)), np.zeros((M, 2 * S), np.uint8)
    n_it = max(F, r)
    lists = np.zeros((n_it, M, S), np.int32)
    det_slot, spawned, dropped = np.full(n, -1, np.int32), np.zeros(n, np.int32), np.full(n, -1, np.int64)
    row = lambda m, s: m * S + s
    new_tracks = []                                     # (s, slot) in spawn order
    for s in range(S):
        rows = np.arange(M) * S + s
        u, v, ok = track_points(prev[rows], cams[s, :9], center)
        ok &= live[rows] != 0
        d4 = det[rows].astype(np.float64)
        with np.errstate(all='ignore'):
            dx, dy = u[:, None] - d4[None, :, 0], v[:, None] - d4[None, :, 1]
            cost = np.sqrt(dx * dx + dy * dy) / (np.float64(res) * d4[None, :, 2])
            adm = ok[:, None] & (valid[rows] != 0)[None, :] & (cost < gate)
        t_idx, d_idx = np.nonzero(adm)
        order = np.lexsort((d_idx, t_idx, cost[t_idx, d_idx]))
        match, det_of = [-1] * M, [-1] * M
        for k in order:
            t, d = t_idx[k], d_idx[k]
            if match[t] < 0 and det_of[d] < 0:
                match[t], det_of[d] = d, t
        for t in range(M):
            i = row(t, s)
            if not live[i]:
                continue
            if match[t] >= 0:
                misses[i] = 0
            else:
                misses[i] += 1
                if misses[i] > max_misses:
                    dropped[i], live[i], ids[i], misses[i] = ids[i], 0, -1, 0
        new = set()
        for d in range(M):
            j = row(d, s)
            if not valid[j]:
                continue
            if det_of[d] >= 0:
                det_slot[j] = det_of[d]
                continue
            free = [t for t in range(M) if not live[row(t, s)]]
            if not free:
                continue
            t = free[0]
            i = row(t, s)
            det_slot[j], live[i], misses[i] = t, 1, 0
            new.add(t)
            work[t, s] = init[j]
            ring[i], count[i] = 0, 0
            new_tracks.append((s, t))
        for t in range(M):
            i = row(t, s)
            spawned[i] = t in new
            go_on = bool(live[i]) and t not in new
            if not live[i]:
                park[i], ids[i] = init[i], -1
                work[t, s] = park[i]
            elif go_on:
                work[t, s] = prev[i]
            work[t, S + s] = work[t, s]
            flags0[t, s] = flags0[t, S + s] = go_on
            L = r if go_on else F
            for it in range(n_it):
                lists[it, t, s] = t * 2 * S + s + (0 if it < L else S)
    for s, t in new_tracks:                              # (sequence, detection) order: slots ascend with detections
        ids[row(t, s)] = next_id[0]
        next_id[0] += 1
    return work.reshape(2 * n, 12), flags0.reshape(-1), lists.reshape(-1), det_slot, spawned, dropped
