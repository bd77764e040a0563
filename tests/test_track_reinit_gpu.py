"""Re-initialising or restarting single sequences of a lockstep tracker on the H100: reset(sequences) / start(poses,
sequences), the mixed step as one captured graph per bucket, its rows against a plain refine step and against
predict_batch, the smoothing restart, the host path, ObjectTracker, and the errors."""
import os

import numpy as np
import pytest
import torch

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


def _frames(frames, t, S):
    return [frames[(t + s) % len(frames)] for s in range(S)]


def _mixed_stages(trk):
    return {k: s for k, s in trk.stages.stages.items() if k[0].startswith('track_mixed')}


def _tracked(e, frames, K, S, steps=2):
    trk = e.tracker(num_sequences=S)
    for t in range(steps):
        trk.step(_frames(frames, t, S), [K] * S)
    return trk


def _check_mixed(e, frames, K, S, reinit, bit_identical_others):
    from gen6d_b200 import track as T
    t = 2
    a, b = _tracked(e, frames, K, S), _tracked(e, frames, K, S)
    ring0, count0 = a._ring.cpu().numpy().copy(), a._count.cpu().numpy().copy()
    prev = a._prev.cpu().numpy().reshape(S, 3, 4).copy()
    a.reset(reinit)
    imgs = _frames(frames, t, S)
    raw, sm, inter = a.step(imgs, [K] * S)
    raw_b, _, inter_b = b.step(imgs, [K] * S)                   # plain refine step from the same previous poses
    others = [s for s in range(S) if s not in reinit]
    F, r = e.cfg['refine_iter'], a.refine_iter
    # keys, shapes, chain lengths
    assert inter['reinit'].tolist() == sorted(reinit) and inter['reinit'].dtype == np.int64
    assert raw.dtype == np.float32 and raw.shape == (S, 3, 4) and sm.dtype == np.float64 and sm.shape == (S, 3, 4)
    assert len(inter['refine_poses']) == 1 + max(F, r) and all(p.shape == (S, 3, 4) for p in inter['refine_poses'])
    assert inter['refine_poses'][0].dtype == np.float64 and np.array_equal(inter['refine_poses'][-1], raw)
    assert inter['bbox_pts'].shape == (S, 8, 2) and inter['smoothed_pts'].shape == (S, 8, 2)
    for k in DET_KEYS:
        assert len(inter[k]) == len(reinit), k
    # rows that kept tracking: the plain refine step's rows
    np.testing.assert_array_equal(inter['refine_poses'][0][others], prev[others])
    d = float(np.abs(raw[others].astype(np.float64) - raw_b[others]).max())
    print(f'S={S} reinit={reinit}: tracked rows vs plain refine step, max |dpose|', d)
    if bit_identical_others:
        assert raw[others].tobytes() == raw_b[others].tobytes()
    else:
        assert d <= 2e-4
    for k in range(r, len(inter['refine_poses'])):
        np.testing.assert_array_equal(inter['refine_poses'][k][others], raw[others])
    # re-initialised rows: predict_batch on their frames at the same batch size
    want_poses, want = e.predict_batch([imgs[s] for s in reinit], [K] * len(reinit))
    if len(reinit) & (len(reinit) - 1) == 0:                 # no padding: detection and selection at the same batch size
        for k in DET_KEYS:
            np.testing.assert_array_equal(inter[k], want[k], err_msg=k)
        np.testing.assert_array_equal(inter['refine_poses'][0][reinit], want['refine_poses'][0])
    else:
        assert inter['sel_ref_idx'].tolist() == want['sel_ref_idx'].tolist()
        np.testing.assert_allclose(inter['refine_poses'][0][reinit], want['refine_poses'][0], atol=1e-4)
    dev = [float(np.abs(inter['refine_poses'][k][reinit].astype(np.float64) - want['refine_poses'][k]).max()) for k in range(F + 1)]
    print('re-initialised rows vs predict_batch, max |dpose| per iteration', dev)
    assert dev[1] < 2e-3
    assert all(dev[k] <= max(2.0 * SENS['gain_R'][k] * 1e-3, 2e-3) for k in range(1, F + 1))
    # smoothing: restarted rows hold one frame, the others continue; the host twin reproduces the step
    count = a._count.cpu().numpy()
    assert (count[reinit] == 1).all() and (count[others] == np.minimum(count0[others] + 1, a.num)).all()
    ring, cnt = ring0.copy(), count0.copy()
    ring[reinit], cnt[reinit] = 0, 0
    want_sm, _ = T.host_smooth(raw, True, a.bbox, np.stack([K] * S), ring, cnt, a.weights)
    assert float(np.abs(want_sm - sm).max() / np.abs(want_sm).max()) <= 1e-12
    np.testing.assert_array_equal(ring, a._ring.cpu().numpy())
    return a


def test_full_reset_and_start_replay_the_existing_graphs(est, video):
    e, _ = est
    frames, K = video
    S = 3
    outs = []
    for seqs in (None, range(S)):
        trk = _tracked(e, frames, K, S)
        trk.reset(seqs) if seqs is not None else trk.reset()
        o1 = trk.step(_frames(frames, 2, S), [K] * S)
        p = TG['track.raw_poses'][:S]
        trk.start(p, seqs) if seqs is not None else trk.start(p)
        o2 = trk.step(_frames(frames, 3, S), [K] * S)
        assert not _mixed_stages(trk) and {k[0] for k in trk.stages.stages} == {'track_full', 'track_refine1'}
        outs.append((o1, o2))
    for (a1, a2), (b1, b2) in [outs]:
        for x, y in ((a1, b1), (a2, b2)):
            assert x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes()
            assert all(np.array_equal(u, v) for u, v in zip(x[2]['refine_poses'], y[2]['refine_poses']))


def test_reset_two_of_four(est, video):
    e, _ = est
    frames, K = video
    _check_mixed(e, frames, K, 4, [1, 3], True)


def test_reset_three_of_four_padded(est, video):
    e, _ = est
    frames, K = video
    trk = _check_mixed(e, frames, K, 4, [0, 1, 3], True)
    assert [k[0] for k in _mixed_stages(trk)] == ['track_mixed4']


def test_one_replay_one_read_and_bucketed_graphs(est, video):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    frames, K = video
    S = 4
    trk = _tracked(e, frames, K, S)
    trk.reset([0])
    trk.step(_frames(frames, 2, S), [K] * S)
    stages = _mixed_stages(trk)
    assert len(stages) == 1
    stage = next(iter(stages.values()))
    trk.reset([2])
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    trk.step(_frames(frames, 3, S), [K] * S)
    assert _mixed_stages(trk) == stages                                   # {2} replays {0}'s graph
    assert REPLAYED_KERNELS[0] - k0 == stage.kernels and IO_BYTES['d2h'] - d0 == stage.static_out[0].numel()
    for m in range(1, S):
        trk.reset(list(range(m)))
        trk.step(_frames(frames, 4 + m, S), [K] * S)
    assert len(_mixed_stages(trk)) <= int(np.ceil(np.log2(S))) + 1


def test_row_flags_on_the_device(est):
    """g6d_glue_refine_problems_rows on the device, unsorted rows with mixed dtype flags: every output row equals, bit for
    bit, that row of g6d_glue_refine_problems_objects launched with that row's flag.  The synthetic object is centred at
    the origin with diameter 2, so its normalisation is the identity and both readings of a pose coincide; the views
    here get a non-trivial normalisation, and poses with digits below float32 resolution, so the flag changes the
    problems (checked)."""
    import ctypes as C
    from gen6d_b200 import _lib, glue, ops
    e, _ = est
    st = e._glue_state()
    v = _lib.GlueViews.from_buffer_copy(st['views'])
    v.norm_scale = 0.7
    for i, x in enumerate((0.11, -0.23, 0.05)):
        v.norm_offset[i] = x
    R, S = st['tables']['ref_num'], 5
    rng = np.random.RandomState(5)
    base = TG['track.raw_poses'][:S].astype(np.float64)
    poses = base + rng.uniform(-0.45, 0.45, base.shape) * np.spacing(np.abs(base).astype(np.float32)).astype(np.float64)
    Ks = np.stack([TG['track.K']] * S, 0)
    frames = torch.zeros(S, 48, 64, 3, dtype=torch.uint8, device='cuda')
    cams, pd = torch.from_numpy(glue.cameras(Ks)).cuda(), torch.from_numpy(poses.reshape(S, 12)).cuda()
    flags = np.array([0, 1, 1, 0, 1], np.uint8)
    idx = np.array([3, 0, 4, 1], np.int32)
    with torch.no_grad():
        got = ops.glue_refine_problems_rows([v], R, S, cams, frames, pd, torch.from_numpy(idx).cuda(), torch.from_numpy(flags).cuda())
        want = {f: ops.glue_refine_problems_objects([v], R, cams, frames, pd, f) for f in (0, 1)}
    torch.cuda.synchronize()
    names = ('jobs', 'que_K', 'que_pose', 'rect', 'ref_Ks', 'ref_poses', 'ref_rows')
    for j, row in enumerate(idx):
        for name, g, w in zip(names, got, want[int(flags[row])]):
            g = g.reshape(len(idx), -1)[j] if name == 'jobs' else g[j]
            w = w.reshape(S, -1)[row] if name == 'jobs' else w[row]
            assert torch.equal(g.reshape(-1).view(torch.uint8), w.reshape(-1).view(torch.uint8)), (j, row, name)
    differ = [not torch.equal(want[0][2][r], want[1][2][r]) or not torch.equal(want[0][3][r], want[1][3][r]) for r in range(S)]
    print('rows whose problem depends on the dtype flag', differ)
    assert any(differ[r] for r in idx)


def test_partial_start_float64_next_to_float32(est, video):
    """A float64 start next to float32 tracked rows (the step is the mixed graph with no re-initialised sequence): the row
    equals, bit for bit, that row of a tracker whose rows were all started in float64, and a single-sequence tracker
    started from the same pose to the lockstep bar."""
    e, _ = est
    frames, K = video
    S = 3
    trk = _tracked(e, frames, K, S)
    prev = trk._prev.cpu().numpy().reshape(S, 3, 4).copy()
    imgs = _frames(frames, 5, S)
    p = TG['track.raw_poses'][4].astype(np.float64)
    p[:, 3] += 0.3 * np.spacing(np.abs(p[:, 3]).astype(np.float32))            # digits below float32 resolution
    trk.start(p[None], [1])
    raw, _, inter = trk.step(imgs, [K] * S)
    assert 'reinit' in inter and inter['reinit'].tolist() == [] and trk._count.cpu().numpy()[1] == 1
    assert [k[0] for k in _mixed_stages(trk)] == ['track_mixed0']
    ref = e.tracker(num_sequences=S)                             # every row started in float64: the float64 refine graph
    ref.start(np.stack([prev[0], p, prev[2]], 0))
    raw_ref = ref.step(imgs, [K] * S)[0]
    assert raw[1].tobytes() == raw_ref[1].tobytes()
    one = e.tracker()
    one.start(p[None])
    want = one.step([imgs[1]], [K])[0][0]
    d = float(np.abs(raw[1].astype(np.float64) - want).max())
    print('partial float64 start next to float32 rows vs a single-sequence tracker, max |dpose|', d)
    assert d <= 2e-4


def test_partial_start_in_any_order(est, video):
    """start(poses, sequences) pairs poses[i] with sequences[i], whatever the order of the list."""
    e, _ = est
    frames, K = video
    S = 3
    P = TG['track.raw_poses'][:S]
    a, b = e.tracker(num_sequences=S), e.tracker(num_sequences=S)
    a.start(P)
    b.start(P[[2, 0]], [2, 0])
    b.start(P[[1]], [1])
    np.testing.assert_array_equal(a._prev, b._prev)                # host state until the first step
    assert a._f32.tolist() == b._f32.tolist()
    imgs = _frames(frames, 1, S)
    ra, sa, _ = a.step(imgs, [K] * S)
    rb, sb, _ = b.step(imgs, [K] * S)
    assert ra.tobytes() == rb.tobytes() and sa.tobytes() == sb.tobytes()


def test_padding_writes_no_real_row(est, video):
    """m = 3 at S = 4 (bucket 4): the padding slot is pointed at a canary frame (another sequence's image) instead of a
    copy of a re-initialised one.  Its detection changes, and every real row's output stays bit-identical: the padding
    reaches no real row."""
    from gen6d_b200 import glue, track as T
    e, _ = est
    frames, K = video
    S, reinit = 4, [0, 1, 3]
    trk = _tracked(e, frames, K, S)
    trk.reset(reinit)
    st = e._glue_state()
    imgs = _frames(frames, 2, S)
    outs = []
    with torch.no_grad():
        dev_frames = e.detector.upload_frame([np.asarray(f) for f in imgs])
        cams = e.detector._to_dev(glue.cameras(np.stack([K] * S, 0)))
        got, b, (seq, tgt, flags, lists) = T._mixed_inputs(S, 1, trk._pending, trk._f32, e.cfg['refine_iter'], trk.refine_iter,
                                                           dev_frames.device)
        assert b == 4 and seq.tolist() == [0, 1, 3, 3]
        canary = seq.clone()
        canary[3] = 2
        fn = trk._mixed_fn(st, b)
        for sq in (seq, canary):
            buf, poses, ring, count = fn(dev_frames, cams, trk._prev.clone(), trk._ring.clone(), trk._count.clone(), sq, tgt, flags, lists)
            outs.append((e.detector._to_host(buf), poses.cpu().numpy(), ring.cpu().numpy(), count.cpu().numpy()))
    (h0, p0, r0, c0), (h1, p1, r1, c1) = outs
    assert p0.tobytes() == p1.tobytes() and r0.tobytes() == r1.tobytes() and c0.tobytes() == c1.tobytes()
    d0, d1 = trk._decode_mixed(h0, got, b), trk._decode_mixed(h1, got, b)
    assert d0[0].tobytes() == d1[0].tobytes() and d0[1].tobytes() == d1[1].tobytes()
    for k in DET_KEYS:
        np.testing.assert_array_equal(d0[2][k], d1[2][k], err_msg=k)
    # the canary did run: the padding slot's detection (row 3 of the packed detections) differs
    n_chain = max(e.cfg['refine_iter'], trk.refine_iter) + 1
    off = n_chain * S * 12 + S * 12 + S * 16 + S * trk.num * 16 + S
    det0, det1 = [h[:off * 8 + b * 32].view(np.float64)[off:].reshape(b, 4) for h in (h0, h1)]
    assert np.array_equal(det0[:3], det1[:3]) and not np.array_equal(det0[3], det1[3])


def test_host_path_matches_graph(est, video):
    e, _ = est
    frames, K = video
    S, reinit = 4, [1, 3]
    outs = []
    for glue_on in (True, False):
        e.cfg['device_glue'] = glue_on
        try:
            trk = e.tracker(num_sequences=S)                          # tracked rows: one step from the same poses
            trk.start(TG['track.raw_poses'][:S])
            trk.reset(reinit)
            outs.append(trk.step(_frames(frames, 2, S), [K] * S))
        finally:
            e.cfg['device_glue'] = True
    (rd, sd, idv), (rh, sh, ih) = outs
    assert idv['reinit'].tolist() == ih['reinit'].tolist() == reinit
    assert np.asarray(idv['sel_ref_idx']).tolist() == np.asarray(ih['sel_ref_idx']).tolist()
    assert len(ih['refine_poses']) == len(idv['refine_poses'])
    others = [0, 2]
    d = float(np.abs(rd[others].astype(np.float64) - rh[others]).max())
    print('mixed step, device graph vs host path, tracked rows max |dpose|', d)
    assert d <= 2e-4
    # the re-initialised rows: predict_batch's device graph against its host path
    dev = [float(np.abs(np.asarray(idv['refine_poses'][k])[reinit].astype(np.float64) - np.asarray(ih['refine_poses'][k])[reinit]).max())
           for k in range(e.cfg['refine_iter'] + 1)]
    print('mixed step, device graph vs host path, re-initialised rows max |dpose| per iteration', dev)
    # the bounds of test_device_glue_prediction_equals_host_path (predict_batch's graph against its host path)
    assert dev[0] < 5e-6 and dev[1] < 2e-4
    assert all(dev[k] <= max(2.0 * SENS['gain_R'][k] * 1e-3, 2e-3) for k in range(1, e.cfg['refine_iter'] + 1))


def test_errors(est, video):
    from gen6d_b200.synthetic import synthetic_database, build_estimator
    e, db = build_estimator()
    frames, K = video
    trk = e.tracker(num_sequences=3)
    for bad in ([3], [-1], [0, 0]):
        with pytest.raises(ValueError):
            trk.reset(bad)
        with pytest.raises(ValueError):
            trk.start(np.zeros((len(bad), 3, 4)), bad)
    with pytest.raises(ValueError):
        trk.start(np.zeros((2, 3, 4)), [1])
    trk.step(frames[:3], [K] * 3)
    trk.reset([1])
    e.build(synthetic_database(seed=8), 'all')
    with pytest.raises(RuntimeError, match='stale'):
        trk.step(frames[:3], [K] * 3)


# ------------------------------------------------------------------------------------------ ObjectTracker
@pytest.fixture(scope='module')
def objs_est():
    from gen6d_b200.synthetic import build_estimator, synthetic_database
    e = build_estimator(synthetic_database(seed=7))[0]
    e.cfg['device_glue'] = True
    dbs = {n: synthetic_database(seed=s) for n, s in (('a', 7), ('b', 8), ('c', 11))}
    return e, dbs


def test_object_tracker_k1_equals_tracker(objs_est, video):
    e, dbs = objs_est
    frames, K = video
    S = 4
    objs = e.object_set()
    objs.add('a', dbs['a'])
    e.build(dbs['a'], 'all')
    ot, tr = objs.tracker(num_sequences=S), e.tracker(num_sequences=S)
    for t in range(2):
        ot.step(_frames(frames, t, S), [K] * S)
        tr.step(_frames(frames, t, S), [K] * S)
    ot.reset([1, 3])
    tr.reset([1, 3])
    got = ot.step(_frames(frames, 2, S), [K] * S)['a']
    want = tr.step(_frames(frames, 2, S), [K] * S)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    for k in DET_KEYS + ('reinit',):
        np.testing.assert_array_equal(got[2][k], want[2][k], err_msg=k)


def test_object_tracker_three_objects_and_kernels(objs_est, video):
    e, dbs = objs_est
    frames, K = video
    S = 2
    objs = e.object_set()
    for n, db in dbs.items():
        objs.add(n, db)
    trk = objs.tracker(num_sequences=S)
    for t in range(2):
        trk.step(_frames(frames, t, S), [K] * S)
    trk.start({n: TG['track.raw_poses'][:S] for n in objs.names})   # every object's tracked row from the same pose
    trk.reset([1])
    imgs = _frames(frames, 2, S)
    got = trk.step(imgs, [K] * S)
    set_pred = objs.predict([imgs[1]], [K])                       # the set's own prediction of the re-initialised frame
    mixed3 = next(iter(_mixed_stages(trk).values())).kernels
    full3 = [s for k, s in trk.stages.stages.items() if k[0] == 'track_full'][0].kernels
    for n, db in dbs.items():
        e.build(db, 'all')
        one = e.tracker(num_sequences=S)
        for t in range(2):
            one.step(_frames(frames, t, S), [K] * S)
        one.start(TG['track.raw_poses'][:S])
        one.reset([1])
        want = one.step(_frames(frames, 2, S), [K] * S)
        d = float(np.abs(got[n][0][0].astype(np.float64) - want[0][0]).max())
        print(f'object {n}: mixed step vs single-object tracker, tracked row max |dpose|', d)
        assert d <= 2e-4
        # the re-initialised row is the set's prediction at the same batch: detection, selection and initial pose bit for
        # bit, then refinements in a refiner batch of K*S rather than K poses (predict_batch vs predict's bounds)
        mine, theirs = got[n][2], set_pred[n][1]
        for k in DET_KEYS + ('det_score',):
            np.testing.assert_array_equal(mine[k], theirs[k], err_msg=(n, k))
        a = np.stack([np.asarray(p, np.float64)[1] for p in mine['refine_poses']])
        c = np.stack([np.asarray(p, np.float64)[0] for p in theirs['refine_poses']])
        dev = np.abs(a - c).reshape(len(a), -1).max(1)
        print(f'object {n}: re-initialised row vs ObjectSet.predict, max |dpose| per iteration', dev)
        assert dev[0] == 0 and dev[1] < 2e-3 and (dev[1:] <= np.maximum(2.0 * SENS['gain_R'][1:len(dev)] * 1e-3, 2e-3)).all()
        # against the single-object tracker the re-initialised row differs by what ObjectSet.predict differs from
        # predict_batch on this frame (the set's one detection GEMM over all objects' kernels): the same initial pose
        single = np.asarray(want[2]['refine_poses'][0], np.float64)[1]
        pb = e.predict_batch([imgs[1]], [K])[1]['refine_poses'][0][0]
        assert np.array_equal(single, pb)
        print(f'object {n}: initial pose, set vs single-object tracker', float(np.abs(a[0] - single).max()),
              '= ObjectSet.predict vs predict_batch', float(np.abs(c[0] - pb).max()))
    # the refinement iterations and the smoothing do not grow with K; only each object's selection does, per gathered
    # frame, as in the full step (which selects on all S frames)
    one_obj = e.object_set()
    one_obj.add('a', dbs['a'])
    t1 = one_obj.tracker(num_sequences=S)
    for t in range(2):
        t1.step(_frames(frames, t, S), [K] * S)
    t1.reset([1])
    t1.step(_frames(frames, 2, S), [K] * S)
    mixed1 = next(iter(_mixed_stages(t1).values())).kernels
    full1 = [s for k, s in t1.stages.stages.items() if k[0] == 'track_full'][0].kernels
    print('mixed-step kernels K=1 / K=3', mixed1, mixed3, 'full-step kernels', full1, full3)
    assert 0 < mixed3 - mixed1 <= full3 - full1
    # a start with differing dtypes and no re-initialisation: the m = 0 mixed graph does not depend on K
    for tk in (trk, t1):
        tk.start({n: TG['track.raw_poses'][5:6].astype(np.float64) for n in tk.names}, [0])
        tk.step(_frames(frames, 3, S), [K] * S)
    k0 = [[s.kernels for k, s in tk.stages.stages.items() if k[0] == 'track_mixed0'] for tk in (trk, t1)]
    # (the refiner stage's launch plan depends on its batch, K*S rows, by a launch or two, as for the refine step)
    assert len(k0[0]) == len(k0[1]) == 1 and abs(k0[0][0] - k0[1][0]) <= 2
