"""Frames of different sizes (gen6d_b200/frames.py, DESIGN.md row f13) on the H100: g6d_frames_canvas against numpy, crops
cut from the canvas against crops of the true-size frame and OpenCV, predict_batch / predict_instances / ObjectSet.predict /
ObjectSet.predict_instances against per-size calls, the four trackers (first steps bit for bit, later steps and partial
re-initialisation), one replay and one read per step, the unchanged single-size path and predict_many."""
import os

import cv2
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENS = np.load(os.path.join(HERE, 'golden', 'sens_golden.npz'))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))
STRICT = ('det_position', 'det_scale_r2q', 'det_que_img')
# crops of a 480x640 frame (y0, x0, h, w): the frame itself, 448x576 and 384x512, principal points shifted to match
CROPS = {'A': (0, 0, 480, 640), 'B': (16, 32, 448, 576), 'C': (48, 64, 384, 512)}


def crop(img, K, which):
    y0, x0, h, w = CROPS[which]
    K = np.array(K, np.float64)
    K[0, 2] -= x0
    K[1, 2] -= y0
    return np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w]), K


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    e, db = build_estimator()
    e.cfg['device_glue'] = True
    return e, db


@pytest.fixture(scope='module')
def mixed(est):
    """Six frames of the database, sizes interleaved A B C A B C."""
    _, db = est
    ids = db.get_img_ids()[:6]
    out = [crop(db.get_image(i), db.get_K(i), 'ABC'[j % 3]) for j, i in enumerate(ids)]
    return [o[0] for o in out], [o[1] for o in out]


def _groups(imgs):
    sizes = [f.shape[:2] for f in imgs]
    return [[i for i in range(len(imgs)) if sizes[i] == z] for z in dict.fromkeys(sizes)]


def _assert_matches_single(got, want, name):
    """tests/test_objects_gpu.py's bars: the selector and refiner batches differ in size, so only split-K summation
    orders change."""
    poses, inter = got
    wposes, winter = want
    np.testing.assert_array_equal(inter['sel_ref_idx'], winter['sel_ref_idx'], err_msg=name)
    np.testing.assert_allclose(inter['det_position'], winter['det_position'], atol=1e-3, err_msg=name)
    np.testing.assert_allclose(inter['det_scale_r2q'], winter['det_scale_r2q'], rtol=1e-4, err_msg=name)
    np.testing.assert_allclose(inter['sel_angle_r2q'], winter['sel_angle_r2q'], atol=1e-4, err_msg=name)
    np.testing.assert_allclose(inter['sel_scores'], winter['sel_scores'], atol=3e-4, err_msg=name)
    a = np.stack([np.asarray(p, np.float64) for p in inter['refine_poses']])
    b = np.stack([np.asarray(p, np.float64) for p in winter['refine_poses']])
    dev = np.abs(a - b).reshape(len(a), -1).max(1)
    print(name, 'mixed sizes vs per-size call, max |dpose| per iteration', dev)
    assert dev[0] < 1e-4, (name, dev)
    assert (dev[1:] <= np.maximum(2.0 * SENS['gain_R'][1:] * 1e-3, 2e-3)).all(), (name, dev)
    np.testing.assert_array_equal(poses, inter['refine_poses'][-1])


def _rows(poses, inter, idx):
    """Rows `idx` (frames) of a prediction's outputs."""
    return poses[idx], {k: ([p[idx] for p in v] if k == 'refine_poses' else v[idx]) for k, v in inter.items()}


def _check_per_size(got, call, imgs, Ks, strict, name):
    poses, inter = got
    for g in _groups(imgs):
        want = call([imgs[i] for i in g], [Ks[i] for i in g])
        mine = _rows(poses, inter, np.asarray(g))
        for k in strict:
            np.testing.assert_array_equal(mine[1][k], want[1][k], err_msg=f'{name} {k} {g}')
        _assert_matches_single(mine, want, f'{name} {g}')


# ------------------------------------------------------------------------------------------ 1. the kernel
def _canvas(packed, table, H, W, out):
    from gen6d_b200 import ops
    host = (ops.FrameEntry * len(table))(*[ops.FrameEntry(o, r, c) for o, r, c in table])
    ops._call('g6d_frames_canvas', ops._p(packed, torch.uint8), packed.numel(), host, len(table), ops._p(out, torch.uint8), H, W,
              ops._stream())


@pytest.mark.parametrize('sizes', [[(7, 13), (5, 9), (7, 13), (1, 1), (3, 17)], [(480, 640), (448, 576), (384, 512)],
                                   [(33, 1)] * 3 + [(2, 40)], [(9, 11)]])
def test_canvas_kernel_equals_numpy(sizes):
    from gen6d_b200 import frames as fr, ops
    rng = np.random.RandomState(len(sizes))
    imgs = [rng.randint(1, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    plan = fr.FramePlan(fr.size_pattern(imgs))
    buf = np.zeros(plan.nbytes, np.uint8)
    for img, (off, _, _) in zip(imgs, plan.table):
        buf[off:off + img.nbytes] = img.reshape(-1)
    packed = torch.from_numpy(buf).cuda()
    want = np.zeros((len(imgs), plan.H, plan.W, 3), np.uint8)
    for i, img in enumerate(imgs):
        want[i, :img.shape[0], :img.shape[1]] = img
    np.testing.assert_array_equal(ops.frames_canvas(packed, plan.table, plan.H, plan.W).cpu().numpy(), want)
    for H, W in ((plan.H, plan.W), (plan.H + 3, plan.W + 130)):                   # a canvas larger than every frame too
        out = torch.full((len(imgs), H, W, 3), 0xA5, dtype=torch.uint8, device='cuda')       # garbage beforehand
        _canvas(packed, plan.table, H, W, out)
        w2 = np.zeros((len(imgs), H, W, 3), np.uint8)
        w2[:, :plan.H, :plan.W] = want
        np.testing.assert_array_equal(out.cpu().numpy(), w2)


def test_canvas_kernel_rejects_bad_tables():
    from gen6d_b200 import _lib, ops
    packed = torch.zeros(300, dtype=torch.uint8, device='cuda')
    for table, H, W in (([(0, 5, 5)], 4, 5), ([(0, 5, 5)], 5, 4), ([(240, 5, 5)], 5, 5), ([(-1, 2, 2)], 5, 5), ([(0, 0, 2)], 5, 5)):
        with pytest.raises(_lib.Gen6DLibraryError, match='g6d_frames_canvas'):
            ops.frames_canvas(packed, table, H, W)


# ------------------------------------------------------------------------------------------ 2. crops from the canvas
def test_crops_from_canvas_equal_true_size_crops_and_opencv(est, mixed):
    from gen6d_b200 import frames as fr, geometry as G, ops
    imgs, _ = mixed
    imgs = imgs[:3]
    plan = fr.FramePlan(fr.size_pattern(imgs))
    buf = np.zeros(plan.nbytes, np.uint8)
    for img, (off, _, _) in zip(imgs, plan.table):
        buf[off:off + img.nbytes] = img.reshape(-1)
    canvas = ops.frames_canvas(torch.from_numpy(buf).cuda(), plan.table, plan.H, plan.W)
    true = [torch.from_numpy(f).cuda() for f in imgs]
    rng = np.random.RandomState(5)
    for i, img in enumerate(imgs):
        h, w = img.shape[:2]
        # windows inside, across the right edge, the bottom edge and the corner, into the canvas padding
        centres = [(w / 2, h / 2), (w - 20, h / 2), (w / 2, h - 15), (w - 10, h - 10), (w + 30, h + 30)]
        for cx, cy in centres:
            size, scale, ang = 128, float(rng.uniform(0.3, 1.5)), float(rng.uniform(-1, 1))
            _, M = G.crop_similarity(None, (cx, cy), scale, ang, size)
            want = cv2.warpAffine(img, M, (size, size), flags=cv2.INTER_LINEAR)
            src = G.affine_dst_to_src(M)
            for s in ((canvas[i].data_ptr(), plan.H, plan.W), G.warp_source(true[i])):
                jobs = torch.from_numpy(G.pack_warp_jobs([s], [src])).cuda()
                np.testing.assert_array_equal(ops.warp_affine_u8(jobs, 1, size, size)[0].cpu().numpy(), want)
            Hm = np.asarray([[scale, 0.1, -cx * scale + 64], [-0.05, scale, -cy * scale + 64], [1e-4, -2e-4, 1.0]])
            want = cv2.warpPerspective(img, Hm, (size, size), flags=cv2.INTER_LINEAR)
            for s in ((canvas[i].data_ptr(), plan.H, plan.W), G.warp_source(true[i])):
                jobs = torch.from_numpy(G.pack_warp_jobs([s], [G.perspective_dst_to_src(Hm)])).cuda()
                np.testing.assert_array_equal(ops.warp_perspective_u8(jobs, 1, size, size)[0].cpu().numpy(), want)


# ------------------------------------------------------------------------------------------ 3-4. predictions
def test_predict_batch_mixed_sizes(est, mixed):
    e, _ = est
    imgs, Ks = mixed
    for sub in ([0, 1, 3, 4], list(range(6))):                         # two sizes, then three
        fi, fk = [imgs[i] for i in sub], [Ks[i] for i in sub]
        got = e.predict_batch(fi, fk)
        assert got[0].shape == (len(sub), 3, 4)
        _check_per_size(got, e.predict_batch, fi, fk, STRICT, f'predict_batch {sub}')


def test_predict_instances_mixed_sizes(est, mixed):
    e, _ = est
    imgs, Ks = mixed
    call = lambda a, b: e.predict_instances(a, b, max_instances=2)
    poses, inter = call(imgs, Ks)
    for g in _groups(imgs):
        wp, want = call([imgs[i] for i in g], [Ks[i] for i in g])
        for k in STRICT + ('det_score', 'instance_valid'):
            np.testing.assert_array_equal(inter[k][g], want[k], err_msg=k)
        np.testing.assert_array_equal(inter['instance_count'][g], want['instance_count'])
        mine = (poses[g], {k: ([p[g] for p in v] if k == 'refine_poses' else v[g]) for k, v in inter.items()})
        _assert_matches_single(mine, (wp, want), f'predict_instances {g}')


@pytest.fixture(scope='module')
def objs(est):
    from gen6d_b200.synthetic import synthetic_database
    e, db = est
    o = e.object_set()
    o.add('a', db)
    o.add('b', synthetic_database(seed=8))
    return o


def test_object_set_predict_mixed_sizes(objs, mixed):
    imgs, Ks = mixed
    res = objs.predict(imgs, Ks)
    for g in _groups(imgs):
        want = objs.predict([imgs[i] for i in g], [Ks[i] for i in g])
        for name in res:
            poses, inter = res[name]
            mine = (poses[g], {k: ([p[g] for p in v] if k == 'refine_poses' else v[g]) for k, v in inter.items()})
            for k in STRICT + ('det_score',):
                np.testing.assert_array_equal(mine[1][k], want[name][1][k], err_msg=f'{name} {k}')
            _assert_matches_single(mine, want[name], f'objs.predict {name} {g}')
    res_i = objs.predict_instances(imgs, Ks, max_instances=2)
    for g in _groups(imgs):
        want = objs.predict_instances([imgs[i] for i in g], [Ks[i] for i in g], max_instances=2)
        for name in res_i:
            poses, inter = res_i[name]
            for k in STRICT + ('det_score', 'instance_valid'):
                np.testing.assert_array_equal(inter[k][g], want[name][1][k], err_msg=f'{name} {k}')
            np.testing.assert_array_equal(inter['instance_count'][g], want[name][1]['instance_count'])
            mine = (poses[g], {k: ([p[g] for p in v] if k == 'refine_poses' else v[g]) for k, v in inter.items()})
            _assert_matches_single(mine, want[name], f'objs.predict_instances {name} {g}')


# ------------------------------------------------------------------------------------------ 5. trackers
@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K']
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _step_frames(video, t, pattern):
    frames, K = video
    out = [crop(frames[(t + s) % len(frames)], K, z) for s, z in enumerate(pattern)]
    return [o[0] for o in out], [o[1] for o in out]


def _one_step(trk, call):
    """call() inside a check that it was one graph replay and one read."""
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    k0, d0, n0 = REPLAYED_KERNELS[0], IO_BYTES['d2h'], dict(trk.stages.stages)
    out = call()
    used = [s for k, s in trk.stages.stages.items() if k not in n0] or None
    # the stage the step replayed: the newly captured one, else the one whose kernels were replayed
    cands = used or [s for s in trk.stages.stages.values() if REPLAYED_KERNELS[0] - k0 == s.kernels]
    assert any(REPLAYED_KERNELS[0] - k0 == s.kernels and IO_BYTES['d2h'] - d0 == s.static_out[0].numel() for s in cands)
    return out


def test_tracker_mixed_sizes(est, video):
    e, _ = est
    pattern, S, T = 'ABAB', 4, 6
    trk = e.tracker(num_sequences=S)
    singles = {z: e.tracker(num_sequences=2) for z in 'AB'}
    rows = {'A': [0, 2], 'B': [1, 3]}
    bar = max(2.0 * float(SENS['gain_R'][1:].max()) * 1e-3, 2e-3)
    for t in range(T):
        imgs, Ks = _step_frames(video, t, pattern)
        raw, sm, inter = _one_step(trk, lambda: trk.step(imgs, Ks))
        for z, r in rows.items():
            wraw, wsm, winter = singles[z].step([imgs[i] for i in r], [Ks[i] for i in r])
            mine = (raw[r], {k: ([p[r] for p in v] if k == 'refine_poses' else v[r]) for k, v in inter.items()
                             if k in STRICT + ('sel_ref_idx', 'sel_angle_r2q', 'sel_scores', 'refine_poses')})
            if t == 0:
                want = e.predict_batch([imgs[i] for i in r], [Ks[i] for i in r])
                for k in STRICT:
                    np.testing.assert_array_equal(mine[1][k], want[1][k], err_msg=k)
                _assert_matches_single(mine, want, f'tracker t=0 {z}')
            # the bar of a whole refinement chain, one more chain's worth per step the deviation is carried
            d, ds = np.abs(raw[r].astype(np.float64) - wraw).max(), np.abs(sm[r] - wsm).max()
            print(f't={t} size {z}: mixed tracker vs single-size tracker, max |dpose| raw {d}, smoothed {ds}')
            assert d <= bar * (1 + t) and ds <= 3 * bar * (1 + t)
    # partial re-initialisation: sequence 1 (size B) re-detected, sequence 2 (size A) restarted from a pose
    trk.reset([1])
    imgs, Ks = _step_frames(video, T, pattern)
    raw, sm, inter = _one_step(trk, lambda: trk.step(imgs, Ks))
    assert inter['reinit'].tolist() == [1]
    want = e.predict_batch([imgs[1]], [Ks[1]])                 # the per-size bucket of size B: one sequence
    for k in STRICT + ('sel_ref_idx',):
        np.testing.assert_array_equal(inter[k], want[1][k], err_msg=k)
    trk.start(TG['track.raw_poses'][:1], [2])
    trk.reset([0, 3])
    imgs, Ks = _step_frames(video, T + 1, pattern)
    raw, sm, inter = _one_step(trk, lambda: trk.step(imgs, Ks))
    assert inter['reinit'].tolist() == [0, 3] and np.isfinite(raw).all()
    for j, s in enumerate((0, 3)):                              # one re-initialised sequence per size: buckets of 1
        want = e.predict_batch([imgs[s]], [Ks[s]])
        for k in STRICT + ('sel_ref_idx',):
            np.testing.assert_array_equal(inter[k][j:j + 1], want[1][k], err_msg=f'{s} {k}')
    keys = [k for k in trk.stages.stages if isinstance(k[0], tuple) and k[0][0][0] == 'track_mixed']
    assert len(keys) == 2 and {k[0][1] for k in keys} == {(0, 1), (1, 1)}
    # a pattern change uses that pattern's graphs
    raw, _, _ = _one_step(trk, lambda: trk.step(*_step_frames(video, T + 2, 'AABB')))
    assert np.isfinite(raw).all()


def test_object_tracker_mixed_sizes(objs, video):
    pattern = 'ABAC'
    imgs, Ks = _step_frames(video, 0, pattern)
    trk = objs.tracker(num_sequences=4)
    out = _one_step(trk, lambda: trk.step(imgs, Ks))
    want = objs.predict(imgs, Ks)
    for name, (raw, sm, inter) in out.items():
        for k in STRICT + ('det_score', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores'):
            np.testing.assert_array_equal(inter[k], want[name][1][k], err_msg=f'{name} {k}')
        for x, y in zip(inter['refine_poses'], want[name][1]['refine_poses']):
            np.testing.assert_array_equal(x, y)
    for t in (1, 2):
        out = _one_step(trk, lambda: trk.step(*_step_frames(video, t, pattern)))
        assert all(np.isfinite(v[0]).all() for v in out.values())
    trk.reset([2])
    out = _one_step(trk, lambda: trk.step(*_step_frames(video, 3, pattern)))
    assert all(v[2]['reinit'].tolist() == [2] for v in out.values())


def _instance_first_step(trk_step, want):
    p, sm, ids, inter = trk_step
    wp, w = want
    valid = w['instance_valid']
    np.testing.assert_array_equal(inter['instance_valid'], valid)
    np.testing.assert_array_equal(p[valid], wp[valid])
    for k in STRICT + ('det_score', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores', 'instance_count'):
        np.testing.assert_array_equal(inter[k], w[k], err_msg=k)
    return ids


def test_instance_trackers_mixed_sizes(est, objs, video):
    e, _ = est
    pattern = 'ABCA'
    imgs, Ks = _step_frames(video, 0, pattern)
    S, M = 4, 2
    trk = e.instance_tracker(num_sequences=S, max_instances=M, gate=1e6, redetect_every=2)
    ids0 = _instance_first_step(_one_step(trk, lambda: trk.step(imgs, Ks)), e.predict_instances(imgs, Ks, max_instances=M))
    _one_step(trk, lambda: trk.step(*_step_frames(video, 1, pattern)))
    _, _, ids1, inter = _one_step(trk, lambda: trk.step(*_step_frames(video, 2, pattern)))      # re-detection
    assert 'det_slot' in inter and inter['dropped'] == []
    live = ids0 >= 0
    np.testing.assert_array_equal(ids1[live], ids0[live])

    otrk = objs.instance_tracker(num_sequences=S, max_instances=M, gate=1e6, redetect_every=2)
    out = _one_step(otrk, lambda: otrk.step(imgs, Ks))
    want = objs.predict_instances(imgs, Ks, max_instances=M)
    ids0 = {n: _instance_first_step(out[n], want[n]) for n in out}
    _one_step(otrk, lambda: otrk.step(*_step_frames(video, 1, pattern)))
    out = _one_step(otrk, lambda: otrk.step(*_step_frames(video, 2, pattern)))
    for n, (_, _, ids1, inter) in out.items():
        assert 'det_slot' in inter and inter['dropped'] == []
        live = ids0[n] >= 0
        np.testing.assert_array_equal(ids1[live], ids0[n][live])


# ------------------------------------------------------------------------------------------ 6. the single-size path
def test_single_size_path_unchanged(est, mixed, monkeypatch):
    from gen6d_b200 import ops
    e, _ = est
    imgs, Ks = mixed
    one = [imgs[i] for i in (0, 3)]
    before = set(e.stages.stages)

    def boom(*a, **k):
        raise AssertionError('g6d_frames_canvas on a single-size batch')
    monkeypatch.setattr(ops, 'frames_canvas', boom)
    e.predict_batch(one, [Ks[0], Ks[3]])
    e.predict_instances(one, [Ks[0], Ks[3]], max_instances=2)
    shapes = (((2, 480, 640, 3), torch.uint8), ((2, 20), torch.float64))
    want = {('predict',) + shapes, (('instances', 2, 1, float(np.float32(0.3)), None),) + shapes}
    assert set(e.stages.stages) - before <= want and want <= set(e.stages.stages)


# ------------------------------------------------------------------------------------------ 7. predict_many
def test_predict_many_groups_by_size(est, mixed):
    e, _ = est
    imgs, Ks = mixed
    res = e.predict_many(imgs, Ks, workers=2, batch=4)
    for g in _groups(imgs):
        pad = g + [g[-1]] * (4 - len(g))
        poses, inter = e.predict_batch([imgs[i] for i in pad], [Ks[i] for i in pad])
        for j, i in enumerate(g):
            np.testing.assert_array_equal(res[i][0], poses[j])
            for k in STRICT + ('sel_ref_idx',):
                np.testing.assert_array_equal(res[i][1][k], inter[k][j], err_msg=k)
