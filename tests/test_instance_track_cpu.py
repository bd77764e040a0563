"""The multi-instance tracker's association (g6d_instances_associate_host: the code the device kernel runs) against the
numpy restatement in instance_assoc_oracle.py, bit for bit on every output, plus its edge cases and argument checks.  No
GPU needed."""
import numpy as np
import pytest

from tests import instance_assoc_oracle as oracle

NUM = 3                 # smoothing ring length of the generated problems
RES = 128.0


def _rotation(rng):
    q = rng.randn(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _project(pose, K, c):
    p = pose[:, :3] @ c + pose[:, 3]
    q = K @ p
    with np.errstate(divide='ignore', invalid='ignore'):
        return q[:2] / q[2]


def make_problem(rng, S=None, M=None, F=None, r=None):
    S = S or int(rng.randint(1, 5))
    M = M or int(rng.choice([1, 2, 3, 4, 5, 8, 16]))
    F = int(rng.randint(0, 5)) if F is None else F
    r = int(rng.randint(1, 5)) if r is None else r
    n = M * S
    center = rng.randn(3) * 0.1
    cams = np.zeros((S, 20))
    for s in range(S):
        f = rng.uniform(300, 800)
        K = np.array([[f, 0, rng.uniform(200, 400)], [0, f * rng.uniform(0.9, 1.1), rng.uniform(150, 300)], [0, 0, 1]])
        cams[s, :9] = K.reshape(-1)
    prev = np.zeros((n, 12))
    for i in range(n):
        pose = np.concatenate([_rotation(rng), np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(2, 8)])[:, None]], 1)
        if rng.rand() < 0.05:
            pose[2, 3] = -pose[2, 3] if rng.rand() < 0.5 else -pose[2, :3] @ center      # behind the camera / depth exactly 0
        prev[i] = pose.reshape(-1)
    live = (rng.rand(n) < rng.uniform(0, 1)).astype(np.int32)
    ids = np.where(live, rng.permutation(max(1000, n))[:n], -1).astype(np.int64)
    max_misses = int(rng.randint(0, 3))
    misses = np.where(live, rng.randint(0, max_misses + 1, n), 0).astype(np.int32)
    det = np.zeros((n, 4), np.float32)
    for i in range(n):
        s = i % S
        t = rng.randint(M) * S + s
        if rng.rand() < 0.7 and prev[t].reshape(3, 4)[2, 3] > 0:   # near some track's projected centre
            xy = _project(prev[t].reshape(3, 4), cams[s, :9].reshape(3, 3), center) + rng.randn(2) * rng.choice([1, 10, 60])
        else:
            xy = rng.uniform(0, 640, 2)
        det[i] = [xy[0], xy[1], 2.0 ** rng.uniform(-1.5, 1.5), rng.randn()]
    if rng.rand() < 0.3:                                              # exact duplicates: cost ties between detections
        a, b = rng.randint(n, size=2)
        det[b % S + S * (b // S)] = det[a]
    if rng.rand() < 0.3 and n > S:                                    # two tracks with one pose: ties between slots
        prev[S + rng.randint(S) if M > 1 else 0] = prev[rng.randint(S)]
    n_valid = rng.randint(0, M + 1, S)
    valid = np.stack([(np.arange(M) < n_valid[s]) for s in range(S)], 1).reshape(-1).astype(np.int32)
    if rng.rand() < 0.2:
        valid = (rng.rand(n) < 0.5).astype(np.int32)                  # not a prefix: the kernel must not assume one
    init = rng.randn(n, 12)
    park = rng.randn(n, 12)
    ring = rng.randn(n, NUM, 8, 2).astype(np.float32)
    count = rng.randint(0, NUM + 1, n).astype(np.int32)
    gate = float(rng.choice([0.05, 0.3, 0.5, 1.0, 3.0]))
    next_id = np.array([rng.randint(0, 5000)], np.int64)
    return dict(det=det, valid=valid, init=init, cams=cams, center=center, res=RES, gate=gate, max_misses=max_misses, F=F, r=r,
                prev=prev, live=live, ids=ids, misses=misses, next_id=next_id, park=park, ring=ring, count=count)


STATE = ('live', 'ids', 'misses', 'next_id', 'park', 'ring', 'count')
OUTS = ('work', 'flags0', 'lists', 'det_slot', 'spawned', 'dropped')


def run_both(p):
    """-> (host twin results, oracle results): dicts of every output and state array."""
    from gen6d_b200.instance_track import host_associate
    res = []
    for fn in (host_associate, oracle.associate):
        q = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
        args = [q[k] for k in ('det', 'valid', 'init', 'cams', 'center', 'res', 'gate', 'max_misses', 'F', 'r', 'prev')]
        outs = fn(*args, *[q[k] for k in STATE])
        res.append({**dict(zip(OUTS, outs)), **{k: q[k] for k in STATE}})
    return res


def assert_same(got, want, tag=''):
    for k in OUTS + STATE:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.shape == w.shape, (tag, k, g.shape, w.shape)
        assert np.array_equal(g.view(np.uint8), w.astype(g.dtype).view(np.uint8)), (tag, k, g, w)


@pytest.fixture(scope='module')
def lib():
    from gen6d_b200.build import build
    build()


def test_random_problems_bit_exact(lib):
    rng = np.random.RandomState(1234)
    n_match = n_spawn = n_drop = n_discard = 0
    for trial in range(2400):
        p = make_problem(rng)
        got, want = run_both(p)
        assert_same(got, want, trial)
        n_spawn += int(got['spawned'].sum())
        n_drop += int((got['dropped'] >= 0).sum())
        n_discard += int(((got['det_slot'] < 0) & (p['valid'] != 0)).sum())
        n_match += int(((got['det_slot'] >= 0) & (got['spawned'][np.maximum(got['det_slot'], 0) * len(p['cams'])
                                                                   + np.arange(len(p['live'])) % len(p['cams'])] == 0)).sum())
    print('matched', n_match, 'spawned', n_spawn, 'dropped', n_drop, 'discarded', n_discard)
    assert min(n_match, n_spawn, n_drop, n_discard) > 50          # every branch is exercised many times


def _simple(S=1, M=3, F=3, r=1, gate=0.5, max_misses=1):
    """A hand-made problem: every slot live at a known pose, detections placed by the caller."""
    rng = np.random.RandomState(0)
    p = make_problem(rng, S=S, M=M, F=F, r=r)
    n = M * S
    p.update(gate=gate, max_misses=max_misses, center=np.zeros(3), live=np.ones(n, np.int32), ids=np.arange(n, dtype=np.int64) + 100,
             misses=np.zeros(n, np.int32), valid=np.ones(n, np.int32), next_id=np.array([7], np.int64))
    K = np.array([500., 0, 320, 0, 500, 240, 0, 0, 1])
    p['cams'][:, :9] = K
    for i in range(n):                                 # slot m of every sequence projects the centre to (100 m + 50, 240)
        m = i // S
        p['prev'][i] = np.array([[1, 0, 0, (100 * m + 50 - 320) * 4 / 500], [0, 1, 0, 0], [0, 0, 1, 4]]).reshape(-1)
    p['det'][:] = [[1000, 1000, 1, 0]]                 # far from everything
    return p


def _place(p, d, x, y=240.0, scale=1.0, s=0):
    p['det'][d * len(p['cams']) + s] = [x, y, scale, 0]


def test_no_live_tracks(lib):
    p = _simple()
    p['live'][:] = 0
    p['ids'][:] = -1
    got, want = run_both(p)
    assert_same(got, want)
    np.testing.assert_array_equal(got['det_slot'], [0, 1, 2])
    np.testing.assert_array_equal(got['ids'], [7, 8, 9])
    assert got['next_id'][0] == 10 and got['spawned'].all()
    np.testing.assert_array_equal(got['work'].reshape(3, 2, 12)[:, 0], p['init'])     # real rows m*2S + s
    np.testing.assert_array_equal(got['ring'], 0)
    np.testing.assert_array_equal(got['count'], 0)


def test_no_valid_detections(lib):
    p = _simple(max_misses=0)
    p['valid'][:] = 0
    p['live'][1] = 0
    p['ids'][1] = -1
    got, want = run_both(p)
    assert_same(got, want)
    assert got['dropped'].tolist() == [100, -1, 102] and not got['live'].any() and (got['ids'] == -1).all()
    np.testing.assert_array_equal(got['park'], p['init'])                # every empty slot parks on its detection row
    np.testing.assert_array_equal(got['det_slot'], -1)
    assert got['next_id'][0] == 7


def test_full_slots_discard_extra_detections(lib):
    p = _simple(gate=0.1)
    got, want = run_both(p)                           # every detection far: no match, one miss each, no free slot
    assert_same(got, want)
    np.testing.assert_array_equal(got['det_slot'], -1)
    np.testing.assert_array_equal(got['misses'], 1)
    np.testing.assert_array_equal(got['ids'], p['ids'])
    assert not got['spawned'].any() and got['next_id'][0] == 7


def test_cost_ties_go_to_lower_slot_then_lower_detection(lib):
    p = _simple(gate=5.0)
    p['prev'][1] = p['prev'][0]                        # slots 0 and 1 at one point
    for d in range(3):
        _place(p, d, 60.0)                             # three identical detections at the same cost from both
    got, want = run_both(p)
    assert_same(got, want)
    np.testing.assert_array_equal(got['det_slot'], [0, 1, 2])          # slot 0 takes det 0, slot 1 det 1, slot 2 det 2
    assert not got['spawned'].any()


def test_cost_at_gate_is_not_admissible(lib):
    p = _simple()
    _place(p, 0, 50.0 - 64.0, scale=1.0)               # about half a box left of slot 0's point
    u, v, _ = oracle.track_points(p['prev'][:1], p['cams'][0, :9], p['center'])
    dx, dy = u[0] - np.float64(p['det'][0, 0]), v[0] - np.float64(p['det'][0, 1])
    cost = np.sqrt(dx * dx + dy * dy) / (np.float64(RES) * np.float64(p['det'][0, 2]))
    assert abs(cost - 0.5) < 1e-9
    p['gate'] = float(cost)                            # the pair's cost exactly
    got, want = run_both(p)
    assert_same(got, want)
    assert got['det_slot'][0] == -1 and got['misses'][0] == 1
    p['gate'] = float(np.nextafter(cost, 1))
    got, want = run_both(p)
    assert_same(got, want)
    assert got['det_slot'][0] == 0 and got['misses'][0] == 0


def test_depth_not_positive_never_matches(lib):
    p = _simple(gate=1e9)
    _place(p, 0, 50.0)
    p['prev'][0, 11] = 0.0                             # depth 0
    p['prev'][1, 11] = -4.0                            # behind the camera
    p['live'][2] = 0
    p['ids'][2] = -1
    got, want = run_both(p)
    assert_same(got, want)
    assert got['misses'][0] == 1 and got['misses'][1] == 1
    np.testing.assert_array_equal(got['det_slot'], [2, -1, -1])        # det 0 spawns in the empty slot 2; dets 1, 2 discarded


def test_max_misses_zero_drops_at_once(lib):
    p = _simple(max_misses=0)
    _place(p, 0, 150.0)                                # slot 1's point
    got, want = run_both(p)
    assert_same(got, want)
    assert got['live'].tolist() == [1, 1, 1] and got['ids'].tolist() == [7, 101, 8]
    assert sorted(i for i in got['dropped'] if i >= 0) == [100, 102]
    np.testing.assert_array_equal(got['det_slot'], [1, 0, 2])
    assert got['spawned'].tolist() == [1, 0, 1]


def test_invalid_rows_never_match(lib):
    p = _simple(gate=5.0)
    for d in range(3):
        _place(p, d, 50.0 + 100 * d)                   # each detection exactly on its slot's point ...
    p['valid'][:] = [0, 1, 0]                          # ... but only detection 1 is valid
    got, want = run_both(p)
    assert_same(got, want)
    np.testing.assert_array_equal(got['det_slot'], [-1, 1, -1])
    np.testing.assert_array_equal(got['misses'], [1, 0, 1])


@pytest.mark.parametrize('F,r', [(1, 3), (2, 2), (3, 1), (0, 2)])
def test_chain_lengths(lib, F, r):
    p = _simple(S=2, F=F, r=r, gate=5.0)
    p['live'][[1, 4]] = 0                              # slot 0 of sequence 1 and slot 2 of sequence 0 are empty
    p['ids'][[1, 4]] = -1
    _place(p, 0, 50.0, s=0)                            # sequence 0: detection 0 matches slot 0
    got, want = run_both(p)
    assert_same(got, want)
    S, M, n_it = 2, 3, max(F, r)
    lists = got['lists'].reshape(n_it, M, S)
    for m in range(M):
        for s in range(S):
            go_on = got['live'][m * S + s] and not got['spawned'][m * S + s]
            L = r if go_on else F
            want_rows = [m * 2 * S + s + (0 if it < L else S) for it in range(n_it)]
            assert lists[:, m, s].tolist() == want_rows, (m, s)
            assert got['flags0'][m * 2 * S + s] == go_on
    work = got['work'].reshape(M, 2 * S, 12)
    np.testing.assert_array_equal(work[:, :S], work[:, S:])           # scratch rows copy the real ones


def test_argument_checks(lib):
    from gen6d_b200 import _lib
    from gen6d_b200.instance_track import check_args
    p = _simple()
    for bad in (dict(gate=0.0), dict(gate=float('inf')), dict(gate=float('nan')), dict(max_misses=-1), dict(F=0, r=0)):
        q = {**p, **bad}
        with pytest.raises(_lib.Gen6DLibraryError):
            run_both(q)
    p17 = make_problem(np.random.RandomState(3), S=1, M=16)
    from gen6d_b200.instance_track import host_associate
    with pytest.raises(_lib.Gen6DLibraryError):          # 17 slots
        host_associate(np.zeros((17, 4), np.float32), np.zeros(17, np.int32), np.zeros((17, 12)), p17['cams'], np.zeros(3), RES, 0.5,
                       1, 1, 1, np.zeros((17, 12)), np.zeros(17, np.int32), np.zeros(17, np.int64), np.zeros(17, np.int32),
                       np.zeros(1, np.int64), np.zeros((17, 12)), np.zeros((17, NUM, 8, 2), np.float32), np.zeros(17, np.int32))
    with pytest.raises(ValueError):                      # state arrays of the wrong dtype are not updated in place
        q = {**p, 'live': p['live'].astype(np.int64)}
        run_both(q)
    good = dict(num_sequences=2, max_instances=4, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1, min_score=None,
                nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5)
    assert check_args(**good)[0] == 4
    for bad in (dict(max_instances=0), dict(max_instances=17), dict(nms_iou=1.5), dict(peak_radius=4), dict(min_score=float('nan')),
                dict(gate=0), dict(gate=-1), dict(gate=float('inf')), dict(gate=float('nan')), dict(max_misses=-1),
                dict(redetect_every=0), dict(num_sequences=0), dict(refine_iter=0), dict(smooth_num=0), dict(smooth_std=0)):
        with pytest.raises(ValueError):
            check_args(**{**good, **bad})
