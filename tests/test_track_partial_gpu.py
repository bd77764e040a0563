"""Partial tracker steps (row f17) on the H100: step(..., sequences=[...]) against a tracker of the bucket's size, the
predict.py smoothing of every stream over its own frames, the relation to the lockstep step, the padding, every frame
kind, drawing, the cost (one replay, one read, one graph per bucket), ObjectTracker and the host path."""
import os

import cv2
import numpy as np
import pytest
import torch

from test_draw_cpu import cv_draw_bbox_3d, nv12_of, project

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))
SENS = np.load(os.path.join(HERE, 'golden', 'sens_golden.npz'))
DET_KEYS = ('det_position', 'det_scale_r2q', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores')


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    e, db = build_estimator()
    e.cfg['device_glue'] = True
    return e, db


@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K']
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _frame(frames, t, s):
    return frames[(t + 3 * s) % len(frames)]


def _state(trk):
    """The tracker's per-sequence state on the host: prev [S,12] (None before any pose), ring, count, pending, f32."""
    prev = None if trk._prev is None else np.asarray(trk._prev.cpu() if isinstance(trk._prev, torch.Tensor) else trk._prev)
    host = lambda a: a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return prev, host(trk._ring).copy(), host(trk._count).copy(), trk._pending.copy(), trk._f32.copy()


def _rows_kept(before, after, idle, K=1, S=None):
    """The idle sequences' state rows (object-major for K objects) keep their bytes."""
    S = S or len(before[3])
    rows = [o * S + s for o in range(K) for s in idle]
    for i, (x, y) in enumerate(zip(before, after)):
        if x is None:
            continue
        r = idle if i >= 3 else rows
        x, y = x.reshape(len(x) if i >= 3 else K * S, -1), y.reshape(len(y) if i >= 3 else K * S, -1)
        assert x[r].tobytes() == y[r].tobytes(), ('prev', 'ring', 'count', 'pending', 'f32')[i]


def _partial_stages(trk):
    return {k: s for k, s in trk.stages.stages.items() if 'rows' in repr(k[0])}


def _same(got, want, where=''):
    if isinstance(want, dict):
        assert set(got) == set(want), (where, sorted(got), sorted(want))
        for k in want:
            _same(got[k], want[k], f'{where}.{k}')
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f'{where}[{i}]')
    elif isinstance(want, torch.Tensor):
        assert torch.equal(got, want), where
    else:
        g, w = np.asarray(got), np.asarray(want)
        assert g.dtype == w.dtype and g.shape == w.shape, where
        assert g.tobytes() == w.tobytes(), where


# ------------------------------------------------------------------------------------------ exactness per step
def _against_bucket_tracker(e, trk, frames, K, seqs, t):
    """One partial step against a fresh tracker of the bucket's size fed the padded frames, started from the partial
    tracker's previous poses for its tracked rows and pending for its re-initialised ones: bit for bit."""
    from gen6d_b200.track import PartialStep
    p = PartialStep(trk.S, 1, seqs, trk._pending, trk._f32, e.cfg['refine_iter'])
    prev = None if trk._prev is None else trk._prev.cpu().numpy().reshape(trk.S, 3, 4)
    imgs = [_frame(frames, t, s) for s in seqs]
    before = _state(trk)
    raw, sm, inter = trk.step(imgs, [K] * len(seqs), sequences=seqs)
    _rows_kept(before, _state(trk), [s for s in range(trk.S) if s not in seqs])
    ref = e.tracker(num_sequences=p.b)
    tracked = [j for j in range(p.b) if not p.pending[j]]
    if tracked:
        ref.start(prev[p.seq[tracked]].astype(np.float32 if p.f32[tracked[0]] else np.float64), tracked)
    r_raw, _, r_inter = ref.step([_frame(frames, t, s) for s in p.seq], [K] * p.b)
    assert raw.tobytes() == r_raw[p.pos].tobytes()
    assert len(inter['refine_poses']) == len(r_inter['refine_poses'])
    for c, rc in zip(inter['refine_poses'], r_inter['refine_poses']):
        assert c.dtype == rc.dtype and c.tobytes() == rc[p.pos].tobytes()
    assert inter['sequences'].tolist() == list(seqs)
    return p, inter


def test_exact_against_a_tracker_of_the_bucket(est, video):
    e, _ = est
    frames, K = video
    S = 4
    trk = e.tracker(num_sequences=S)
    p, inter = _against_bucket_tracker(e, trk, frames, K, [1, 3], 0)             # full, b = 2
    assert p.kind == 'full' and 'det_position' in inter and trk._pending.tolist() == [True, False, True, False]
    p, _ = _against_bucket_tracker(e, trk, frames, K, [0, 1, 2], 1)             # mixed (0, 2 pending), padded to 4
    assert p.kind == 'mixed' and p.b == 4
    p, _ = _against_bucket_tracker(e, trk, frames, K, [3, 0], 2)                # refine, b = 2
    assert p.kind == 'refine'
    p, _ = _against_bucket_tracker(e, trk, frames, K, [2, 3, 1], 3)             # refine, padded to 4
    assert p.kind == 'refine' and p.b == 4
    trk.reset([1])
    p, inter = _against_bucket_tracker(e, trk, frames, K, [1, 2, 0], 4)         # mixed with a reset, padded to 4
    assert p.kind == 'mixed' and inter['reinit'].tolist() == [1] and len(inter['sel_ref_idx']) == 1
    p, _ = _against_bucket_tracker(e, trk, frames, K, [2], 5)                   # refine, b = 1
    assert not trk._pending.any()


# ------------------------------------------------------------------------------------------ a schedule
def _events(S):
    """Before tick t: ('reset', s) or ('start', s, pose) of a sequence."""
    return {5: ('reset', 2), 8: ('start', 0, TG['track.raw_poses'][3]), 10: ('reset', 3)}


def _schedule(S, T, seed):
    """Seeded activity: per tick the active sequences (each with p = 0.6, at least one), in a random order.  A sequence
    reset or started before tick t sits that tick out and is listed at t + 1 (it stays pending, or keeps its start pose,
    while idle)."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(T):
        act = np.flatnonzero(rng.rand(S) < 0.6)
        if not len(act):
            act = rng.randint(0, S, 1)
        out.append(rng.permutation(act).tolist())
    for t, ev in _events(S).items():
        s = ev[1]
        out[t] = [q for q in out[t] if q != s] or [(s + 1) % S]
        out[t + 1] = [q for q in out[t + 1] if q != s] + [s]
    return out


def _run_schedule(trk, frames, K, sched, events, check=None, **kw):
    outs = []
    for t, seqs in enumerate(sched):
        ev = events.get(t)
        if ev and ev[0] == 'reset':
            trk.reset([ev[1]])
        elif ev:
            trk.start(ev[2][None], [ev[1]])
        before = _state(trk) if check else None
        res = trk.step([_frame(frames, t, s) for s in seqs], [K] * len(seqs), sequences=seqs, **kw)
        if check:
            check(before, _state(trk), [s for s in range(trk.S) if s not in seqs])
        outs.append(res)
    return outs


def test_schedule_smooths_every_stream_over_its_own_frames(est, video):
    from gen6d_b200 import track as T
    e, _ = est
    frames, K = video
    S, sched, events = 4, _schedule(4, 14, 3), _events(4)
    trk = e.tracker(num_sequences=S)
    outs = _run_schedule(trk, frames, K, sched, events, check=_rows_kept)
    ring, count = np.zeros((S, trk.num, 8, 2), np.float32), np.zeros(S, np.int32)
    worst = 0.0
    for t, (seqs, (raw, sm, inter)) in enumerate(zip(sched, outs)):
        ev = events.get(t)
        if ev:
            ring[ev[1]], count[ev[1]] = 0, 0
        for i, s in enumerate(seqs):
            r, c = ring[s:s + 1], count[s:s + 1]                                   # views: updated in place
            want_sm, want_avg = T.host_smooth(raw[i:i + 1], True, trk.bbox, K[None], r, c, trk.weights)
            assert inter['bbox_pts'][i].tobytes() == r[0, c[0] - 1].astype(np.float32).tobytes(), (t, s)
            assert inter['smoothed_pts'][i].tobytes() == want_avg[0].tobytes(), (t, s)
            worst = max(worst, float(np.abs(want_sm[0] - sm[i]).max() / np.abs(want_sm).max()))
    print('partial schedule: smoothed poses vs host_smooth over each stream, max relative |d|', worst)
    assert worst <= 1e-9
    np.testing.assert_array_equal(ring, trk._ring.cpu().numpy())
    np.testing.assert_array_equal(count, trk._count.cpu().numpy())
    # the started sequence refined from its start pose at its next listed step; the reset ones were re-initialised then
    first = outs[9][2]['refine_poses'][0][sched[9].index(0)]
    np.testing.assert_array_equal(first, TG['track.raw_poses'][3].astype(first.dtype))
    assert outs[6][2]['reinit'].tolist() == [2] and outs[11][2]['reinit'].tolist() == [3]


# ------------------------------------------------------------------------------------------ relation to lockstep
def test_all_sequences_replay_the_lockstep_graphs(est, video):
    e, _ = est
    frames, K = video
    S = 3
    a, b, c = (e.tracker(num_sequences=S) for _ in range(3))
    perm = [2, 0, 1]
    for t in range(3):
        if t == 2:
            for trk in (a, b, c):
                trk.reset([1])
        imgs = [_frame(frames, t, s) for s in range(S)]
        ra = a.step(imgs, [K] * S)
        rb = b.step(imgs, [K] * S, sequences=list(range(S)))
        rc = c.step([imgs[s] for s in perm], [K] * S, sequences=perm)
        assert rb[2].pop('sequences').tolist() == [0, 1, 2] and rc[2].pop('sequences').tolist() == perm
        _same(rb, ra, f'ascending {t}')
        inv = np.argsort(perm)
        _same((rc[0][inv], rc[1][inv]), (ra[0], ra[1]), f'permuted {t}')
        for k, v in ra[2].items():
            if k == 'reinit' or (t == 2 and k in DET_KEYS):                        # per re-initialised sequence, ascending
                _same(rc[2][k], v, f'permuted {t} {k}')
            elif k == 'refine_poses':
                _same([x[inv] for x in rc[2][k]], v, f'permuted {t} {k}')
            else:
                _same(np.asarray(rc[2][k])[inv], v, f'permuted {t} {k}')
    assert set(a.stages.stages) == set(b.stages.stages) == set(c.stages.stages) and not _partial_stages(b)


def test_single_sequence_within_the_lockstep_bar(est, video):
    e, _ = est
    frames, K = video
    S = 4
    trk = e.tracker(num_sequences=S)
    for t in range(2):
        trk.step([_frame(frames, t, s) for s in range(S)], [K] * S)
    prev = trk._prev.cpu().numpy().reshape(S, 3, 4)
    raw = trk.step([_frame(frames, 2, 2)], [K], sequences=[2])[0]
    one = e.tracker()
    one.start(prev[2:3].astype(np.float32))
    want = one.step([_frame(frames, 2, 2)], [K])[0]
    d = float(np.abs(raw.astype(np.float64) - want).max())
    print('partial step of one sequence vs a num_sequences=1 tracker, max |dpose|', d)
    assert d <= 2e-4


# ------------------------------------------------------------------------------------------ padding canary
@pytest.mark.parametrize('kind', ['refine', 'full'])
def test_padding_writes_no_real_row(est, video, kind):
    """Three of four sequences (bucket 4): the padding slot is pointed at another stream's frame instead of a copy of the
    last listed one.  The tracker state the graph body returns and every real row of its results stay bit-identical."""
    from gen6d_b200 import glue
    from gen6d_b200.track import PartialStep, _compact_fn
    e, _ = est
    frames, K = video
    S, seqs = 4, [0, 1, 3]
    trk = e.tracker(num_sequences=S)
    if kind == 'refine':
        trk.step([_frame(frames, 0, s) for s in range(S)], [K] * S)
    p = PartialStep(S, 1, seqs, trk._pending, trk._f32, e.cfg['refine_iter'])
    assert p.kind == kind and p.b == 4 and p.seq.tolist() == [0, 1, 3, 3]
    st = e._glue_state()
    trk._to(True)
    prev = trk._prev if trk._prev is not None else torch.zeros(S, 12, dtype=torch.float64, device='cuda')
    fn = _compact_fn(trk._full_fn(st) if kind == 'full' else trk._refine_fn(st, True), kind == 'full')
    outs = []
    with torch.no_grad():
        for last in (3, 2):                                  # the padding copy, then the canary
            imgs = [_frame(frames, 1, s) for s in (0, 1, 3, last)]
            cams = e.detector._to_dev(glue.cameras(np.stack([K] * 4, 0)))
            buf, p2, r2, c2 = fn(e.detector.upload_frame(imgs), cams, prev.clone(), trk._ring.clone(), trk._count.clone(),
                                 *p.graph_inputs('cuda'))
            outs.append((e.detector._to_host(buf), p2.cpu().numpy(), r2.cpu().numpy(), c2.cpu().numpy()))
    (h0, *s0), (h1, *s1) = outs
    assert all(x.tobytes() == y.tobytes() for x, y in zip(s0, s1))
    d0, d1 = (p.results(*trk._decode(h, kind == 'full', True, S=4)) for h in (h0, h1))
    _same(d0, d1, 'real rows')
    if kind == 'full':                                       # the canary did run: the padding slot's detection differs
        full = [trk._decode(h, True, True, S=4)[2] for h in (h0, h1)]
        assert not np.array_equal(full[0]['det_position'][3], full[1]['det_position'][3])


# ------------------------------------------------------------------------------------------ inputs and drawing
def _inputs(kind, imgs):
    """The listed frames as `kind`, and the RGB frames the graph holds (numpy) for the reference run."""
    from gen6d_b200.frames import NV12, Resized
    if kind == 'numpy':
        return imgs, imgs
    if kind == 'cuda':
        return [torch.from_numpy(im).cuda() for im in imgs], imgs
    if kind == 'nv12':
        ins, ref = [], []
        for im in imgs:
            y, uv = nv12_of(im)
            ins.append(NV12(torch.from_numpy(y).cuda(), torch.from_numpy(uv).cuda()))
            ref.append(cv2.cvtColor(np.vstack([y, uv]), cv2.COLOR_YUV2RGB_NV12))
        return ins, ref
    if kind == 'resized':                                    # a 2x source resized to the working size on the device
        ins, ref = [], []
        for im in imgs:
            h, w = im.shape[:2]
            big = np.ascontiguousarray(np.repeat(np.repeat(im, 2, 0), 2, 1))
            ins.append(Resized(torch.from_numpy(big).cuda(), size=(h, w)))
            ref.append(cv2.resize(big, (w, h), interpolation=cv2.INTER_LINEAR))
        return ins, ref
    raise ValueError(kind)


SCHED = [[0, 2, 3], [1, 2], [3, 0], [2], [0, 1, 2, 3], [1, 3, 0]]


def _two_sizes(imgs, seqs):
    """Odd sequences' frames cropped to a smaller size (a top-left crop keeps K)."""
    return [np.ascontiguousarray(im[:400, :560]) if s % 2 else im for im, s in zip(imgs, seqs)]


@pytest.mark.parametrize('kind', ['cuda', 'nv12', 'resized', 'two_sizes'])
def test_frame_kinds_equal_the_numpy_path(est, video, kind):
    e, _ = est
    frames, K = video
    S = 4
    a, b = e.tracker(num_sequences=S), e.tracker(num_sequences=S)
    for t, seqs in enumerate(SCHED):
        imgs = [np.ascontiguousarray(_frame(frames, t, s)) for s in seqs]
        if kind == 'two_sizes':
            imgs = _two_sizes(imgs, seqs)
            ins, ref = [torch.from_numpy(im).cuda() for im in imgs], imgs
        else:
            ins, ref = _inputs(kind, imgs)
        got = a.step(ins, [K] * len(seqs), sequences=seqs)
        want = b.step(ref, [K] * len(seqs), sequences=seqs)
        _same(got, want, f'{kind} step {t}')


def test_drawing_and_destinations(est, video):
    """draw='smoothed': the drawn frames of the listed sequences are draw_bbox_3d with the step's own poses, results equal a
    non-drawing tracker's, out= buffers of idle sequences keep their bytes, and new buffers replay the same graphs."""
    e, _ = est
    frames, _ = video
    K = TG['track.K'].astype(np.float32)
    S = 4
    dt, nt = e.tracker(num_sequences=S, draw='smoothed'), e.tracker(num_sequences=S)
    h, w = frames[0].shape[:2]
    for t, seqs in enumerate(SCHED):
        imgs = [np.ascontiguousarray(_frame(frames, t, s)) for s in seqs]
        raw, sm, inter = dt.step(imgs, [K] * len(seqs), sequences=seqs)
        want = nt.step(imgs, [K] * len(seqs), sequences=seqs)
        drawn = inter.pop('drawn')['smoothed']
        _same((raw, sm, inter), want, f'step {t}')
        assert len(drawn) == len(seqs)
        for i in range(len(seqs)):
            np.testing.assert_array_equal(drawn[i].cpu().numpy(), cv_draw_bbox_3d(imgs[i], project(dt.bbox, sm[i], K), (0, 0, 255)))
    n = len(dt.stages.stages)
    for t, seqs in enumerate([[3, 0], [2], [1, 3, 0]] * 2):      # refine steps of buckets 2, 1 and 4 (padded), new buffers
        bufs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda') for _ in range(S)]
        keep = [x.clone() for x in bufs]
        imgs = [np.ascontiguousarray(_frame(frames, 10 + t, s)) for s in seqs]
        raw, sm, inter = dt.step(imgs, [K] * len(seqs), out={'smoothed': [bufs[s] for s in seqs]}, sequences=seqs)
        assert 'drawn' not in inter
        for s in range(S):
            if s in seqs:
                i = seqs.index(s)
                np.testing.assert_array_equal(bufs[s].cpu().numpy(), cv_draw_bbox_3d(imgs[i], project(dt.bbox, sm[i], K), (0, 0, 255)))
            else:
                assert torch.equal(bufs[s], keep[s]), (t, s)
    assert len(dt.stages.stages) == n


# ------------------------------------------------------------------------------------------ cost
def test_one_replay_one_read_one_graph_per_bucket(est, video):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    frames, K = video
    S = 10
    trk = e.tracker(num_sequences=S)
    trk.step([_frame(frames, 0, s) for s in range(S)], [K] * S)
    rng = np.random.RandomState(4)
    seen = {}
    for t in range(12):
        a = [1, 2, 3, 4, 5, 7, 9][t % 7]
        seqs = rng.permutation(S)[:a].tolist()
        k0, d0, n0 = REPLAYED_KERNELS[0], IO_BYTES['d2h'], dict(_partial_stages(trk))
        trk.step([_frame(frames, t, s) for s in seqs], [K] * a, sequences=seqs)
        stages = _partial_stages(trk)
        new = set(stages) - set(n0)
        (key,) = [k for k in stages if k[0][2] == min(S, 1 << (a - 1).bit_length())]
        st = stages[key]
        assert REPLAYED_KERNELS[0] - k0 == st.kernels and IO_BYTES['d2h'] - d0 == st.static_out[0].numel()
        assert not new or (new == {key} and key not in seen)
        seen[key] = st
    assert len(_partial_stages(trk)) == len(seen) == 5                      # buckets 1, 2, 4, 8 and 10 (capped at S)
    print('refine graphs per bucket, kernels', {k[0][2]: s.kernels for k, s in seen.items()})


# ------------------------------------------------------------------------------------------ objects and the host path
@pytest.fixture(scope='module')
def objs_est():
    from gen6d_b200.synthetic import build_estimator, synthetic_database
    e = build_estimator(synthetic_database(seed=7))[0]
    e.cfg['device_glue'] = True
    dbs = {n: synthetic_database(seed=s) for n, s in (('a', 7), ('b', 8))}
    return e, dbs


def test_object_tracker(objs_est, video):
    e, dbs = objs_est
    frames, K = video
    S, sched, events = 4, _schedule(4, 12, 5), _events(4)
    objs = e.object_set()
    objs.add('a', dbs['a'])
    e.build(dbs['a'], 'all')
    ot, tr = objs.tracker(num_sequences=S), e.tracker(num_sequences=S)
    ev1 = {t: (v if v[0] == 'reset' else ('start', v[1], {'a': v[2][None]})) for t, v in events.items()}
    got, want = [], _run_schedule(tr, frames, K, sched, events)
    for t, seqs in enumerate(sched):                           # ObjectTracker.start takes {name: poses}
        ev = ev1.get(t)
        if ev and ev[0] == 'reset':
            ot.reset([ev[1]])
        elif ev:
            ot.start(ev[2], [ev[1]])
        before = _state(ot)
        got.append(ot.step([_frame(frames, t, s) for s in seqs], [K] * len(seqs), sequences=seqs)['a'])
        _rows_kept(before, _state(ot), [s for s in range(S) if s not in seqs])
    for t, (g, w) in enumerate(zip(got, want)):
        g[2].pop('det_score', None)
        _same(g, w, f'K=1 step {t}')
    # K = 2 over the same schedule: shapes, and the idle rows of both objects untouched
    objs.add('b', dbs['b'])
    o2 = objs.tracker(num_sequences=S)
    for t, seqs in enumerate(sched):
        ev = ev1.get(t)
        if ev and ev[0] == 'reset':
            o2.reset([ev[1]])
        elif ev:
            o2.start({n: ev[2]['a'] for n in o2.names}, [ev[1]])
        before = _state(o2)
        res = o2.step([_frame(frames, t, s) for s in seqs], [K] * len(seqs), sequences=seqs)
        _rows_kept(before, _state(o2), [s for s in range(S) if s not in seqs], K=2, S=S)
        for n in o2.names:
            assert res[n][0].shape == (len(seqs), 3, 4) and res[n][2]['sequences'].tolist() == seqs


def test_host_path_matches_graph(est, video):
    """Each case one partial step from the same start poses (a refine step, a mixed one after a reset, padded, a single
    sequence, every sequence), on the graph and on the host path: the bar of test_host_path_matches_graph."""
    e, _ = est
    frames, K = video
    S = 4
    cases = [([2, 0], []), ([1, 3, 2], [1]), ([3], []), ([0, 1, 2, 3], [2])]
    for t, (seqs, reinit) in enumerate(cases):
        outs = []
        for glue_on in (True, False):
            e.cfg['device_glue'] = glue_on
            try:
                trk = e.tracker(num_sequences=S)
                trk.start(TG['track.raw_poses'][:S])
                if reinit:
                    trk.reset(reinit)
                before = _state(trk)
                outs.append(trk.step([_frame(frames, t, s) for s in seqs], [K] * len(seqs), sequences=seqs))
                _rows_kept(before, _state(trk), [s for s in range(S) if s not in seqs])
            finally:
                e.cfg['device_glue'] = True
        (rd, _, idv), (rh, _, ih) = outs
        assert idv['sequences'].tolist() == ih['sequences'].tolist() == seqs
        assert idv.get('reinit', np.zeros(0)).tolist() == ih.get('reinit', np.zeros(0)).tolist() == reinit
        tracked = [i for i, s in enumerate(seqs) if s not in reinit]
        d = float(np.abs(rd[tracked].astype(np.float64) - rh[tracked]).max())
        print(f'case {seqs}: tracked rows, device graph vs host path, max |dpose|', d)
        assert d <= 2e-4
        if reinit:
            i = [seqs.index(s) for s in reinit]
            assert np.asarray(idv['sel_ref_idx']).tolist() == np.asarray(ih['sel_ref_idx']).tolist()
            dev = [float(np.abs(np.asarray(idv['refine_poses'][k])[i].astype(np.float64) - np.asarray(ih['refine_poses'][k])[i]).max())
                   for k in range(e.cfg['refine_iter'] + 1)]
            print(f'case {seqs}: re-initialised rows, device graph vs host path, max |dpose| per iteration', dev)
            assert dev[0] < 5e-6 and dev[1] < 2e-4
            assert all(dev[k] <= max(2.0 * SENS['gain_R'][k] * 1e-3, 2e-3) for k in range(1, e.cfg['refine_iter'] + 1))
