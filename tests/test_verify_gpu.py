"""Checking tracked poses with the detector (row f20) on the H100: g6d_verify_windows / g6d_verify_judge against their
host twins; Gen6DEstimator.verify_poses against an oracle built from existing parts (the twin's records, windows cut
with cv2.warpAffine, the detector on that batch, the judge's twin) for numpy, CUDA RGB, NV12, Resized and two-size
frames; the verifying trackers against trackers without verification, bit for bit, with the schedule, the records and
the reset policy; objects against single-object estimators."""
import cv2
import numpy as np
import pytest
import torch

from gen6d_b200 import frames as fr, geometry as G, glue, ops, verify as V

pytestmark = pytest.mark.gpu
W = 256


def _same(got, want, where=''):
    if isinstance(want, dict):
        assert set(got) == set(want), (where, set(got) ^ set(want))
        for k in want:
            _same(got[k], want[k], f'{where}.{k}')
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f'{where}[{i}]')
    else:
        g, w = np.asarray(got), np.asarray(want)
        assert g.dtype == w.dtype and g.shape == w.shape, (where, g.dtype, w.dtype, g.shape, w.shape)
        np.testing.assert_array_equal(g, w, err_msg=where)


def _without_verify(res):
    raw, smoothed, inter = res
    return raw, smoothed, {k: v for k, v in inter.items() if k != 'verify'}


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    e, db = build_estimator()
    e.cfg['device_glue'] = True
    return e, db


@pytest.fixture(scope='module')
def frames(est):
    _, db = est
    ids = db.get_img_ids()[:4]
    return [np.ascontiguousarray(db.get_image(i)) for i in ids], [db.get_K(i) for i in ids]


@pytest.fixture(scope='module')
def poses(est, frames):
    """predict_batch's poses on the frames, one pushed behind the camera."""
    e, _ = est
    p, _ = e.predict_batch(*frames)
    p = p.copy()
    p[2, :, 3] *= -1
    return p


# ------------------------------------------------------------------------------------------ kernels
def test_kernels_equal_their_host_twins(est, frames, poses):
    e, db = est
    rng = np.random.RandomState(0)
    _, Ks = frames
    refs_np = [glue.selector_refs(e.ref_info), glue.selector_refs({**e.ref_info, 'center': e.ref_info['center'] + 0.01})]
    keep = [{k: torch.from_numpy(np.ascontiguousarray(r[k])).cuda() for k in ('poses', 'cen', 'f', 'dist')} for r in refs_np]
    structs = [glue.refs_struct({**{k: t.data_ptr() for k, t in d.items()}, 'center': r['center']}) for d, r in zip(keep, refs_np)]
    cams = glue.cameras(np.stack(Ks, 0))
    P = np.concatenate([poses, poses + rng.randn(*poses.shape) * 0.01], 0)
    P[5, 0, 0] = np.nan
    for f32 in (False, True):
        p = P.astype(np.float32) if f32 else P
        got = ops.verify_windows(structs, torch.from_numpy(cams).cuda(), torch.from_numpy(p.astype(np.float64).reshape(-1, 12)).cuda(), f32)
        _same(got.cpu().numpy(), V.host_windows(p, f32, refs_np, cams), f'windows f32={f32}')
    n = 64
    rec = np.stack([rng.rand(n) * 640, rng.rand(n) * 480, 0.3 + rng.rand(n) * 2, (rng.rand(n) > 0.2)], 1).astype(np.float32)
    det = np.stack([rng.rand(n) * 256, rng.rand(n) * 256, rng.rand(n) * 3, rng.randn(n)], 1).astype(np.float32)
    det[4, 3] = np.nan
    for thr in [(None, None), (0.0, None), (None, 0.3), (0.5, 0.2), (np.inf, None)]:
        out, lost = ops.verify_judge(torch.from_numpy(rec).cuda(), torch.from_numpy(det).cuda(), W, 128, *thr)
        want = V.host_judge(rec, det, W, 128, *thr)
        _same((out.cpu().numpy(), lost.cpu().numpy()), want, f'judge {thr}')


# ------------------------------------------------------------------------------------------ verify_poses
def oracle_verify(e, imgs, Ks, poses, lost_score=None, lost_gate=None, refs=None, detector=None):
    """The twin's records, windows cut with cv2.warpAffine, the detector on them, the judge's twin -> (result, windows)."""
    f32 = poses.dtype == np.float32
    refs = refs or glue.selector_refs(e.ref_info)
    rec = V.host_windows(poses, f32, [refs], glue.cameras(np.stack([np.asarray(K) for K in Ks], 0)))
    wins = np.stack([G.crop_similarity(img, rec[i, :2], 1 / rec[i, 2], 0, W)[0] for i, img in enumerate(imgs)], 0)
    with torch.no_grad():
        det = (detector or e.detector._detect_u8)(torch.from_numpy(wins).cuda()).cpu().numpy()
    out, lost = V.host_judge(rec, det, W, e.cfg['ref_resolution'], lost_score, lost_gate)
    return {'position': out[:, :2], 'scale': out[:, 2], 'score': out[:, 3], 'offset': out[:, 4], 'lost': lost != 0,
            'window_center': rec[:, :2], 'window_scale': rec[:, 2]}, wins, rec


def test_device_windows_equal_cv2(est, frames, poses):
    e, _ = est
    imgs, Ks = frames
    _, wins, rec = oracle_verify(e, imgs, Ks, poses)
    dev = torch.from_numpy(np.stack(imgs, 0)).cuda()
    got = ops.warp_affine_u8(ops.glue_detection_jobs(torch.from_numpy(rec).cuda(), dev, W), len(imgs), W, W)
    _same(got.cpu().numpy(), wins, 'windows')


def _nv12(img):
    h, w = img.shape[:2]
    i420 = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    yuv = np.vstack([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])
    surf = torch.from_numpy(yuv).cuda()
    return fr.NV12(surf[:h], surf[h:]), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)


@pytest.mark.parametrize('form', ['numpy', 'cuda', 'nv12', 'resized', 'two_sizes'])
@pytest.mark.parametrize('thr', [(None, None), (0.0, 0.3)])
def test_verify_poses_equals_the_oracle(est, frames, poses, form, thr):
    e, _ = est
    imgs, Ks = frames
    Ks = [np.asarray(K, np.float64) for K in Ks]
    if form == 'cuda':
        dev, ref = [torch.from_numpy(i).cuda() for i in imgs], imgs
    elif form == 'nv12':
        pairs = [_nv12(i) for i in imgs]
        dev, ref = [p[0] for p in pairs], [p[1] for p in pairs]
    elif form == 'resized':
        dev = [fr.Resized(torch.from_numpy(i).cuda(), size=(360, 480)) for i in imgs]
        ref = [cv2.resize(i, (480, 360), interpolation=cv2.INTER_LINEAR) for i in imgs]
        Ks = [f.intrinsics(K) for f, K in zip(dev, Ks)]
    elif form == 'two_sizes':
        ref = [i if j % 2 else np.ascontiguousarray(i[16:464, 32:608]) for j, i in enumerate(imgs)]
        Ks = [K if j % 2 else K - np.asarray([[0, 0, 32], [0, 0, 16], [0, 0, 0]]) for j, K in enumerate(Ks)]
        dev = ref
    else:
        dev = ref = imgs
    for p in (poses.astype(np.float64), poses.astype(np.float32)):
        got = e.verify_poses(dev, Ks, p, *thr)
        want, _, _ = oracle_verify(e, ref, Ks, p, *thr)
        _same(got, want, f'{form} {p.dtype}')
        assert got['lost'][2]                                         # behind the camera


def test_verify_poses_is_one_graph_and_one_read(est, frames, poses):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    imgs, Ks = frames
    e.verify_poses(imgs, Ks, poses, lost_score=1.0)
    name = ('verify_poses', int(poses.dtype == np.float32), 1.0, None)
    stage = e.stages.stages[next(k for k in e.stages.stages if k[0] == name)]
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    e.verify_poses(imgs, Ks, poses, lost_score=1.0)
    assert REPLAYED_KERNELS[0] - k0 == stage.kernels and IO_BYTES['d2h'] - d0 == stage.static_out.numel() * 8


# ------------------------------------------------------------------------------------------ trackers
@pytest.fixture(scope='module')
def video(est):
    """12 steps x 3 sequences: sequence s at step t sees view (3*t + 5*s) % 72 of the database."""
    _, db = est
    ids = db.get_img_ids()
    return [[(np.ascontiguousarray(db.get_image(ids[(3 * t + 5 * s) % len(ids)])), db.get_K(ids[(3 * t + 5 * s) % len(ids)]))
             for s in range(3)] for t in range(12)]


# (sequences stepped, reset before the step); verify_every = 3 verifies at steps 3, 6 and 9
PLAN = [(None, None), (None, None), (None, None), (None, None), (None, [1]), ([0, 2], None), ([2, 0], None), ([1], None),
        (None, None), (None, None), ([1, 2], None), (None, None)]


def _run(trk, video, plan, on_step=None):
    out = []
    for t, (seqs, reset) in enumerate(plan):
        if reset is not None:
            trk.reset(reset)
        rows = range(3) if seqs is None else seqs
        imgs, Ks = [video[t][s][0] for s in rows], [video[t][s][1] for s in rows]
        out.append(trk.step(imgs, Ks, sequences=seqs))
        if on_step:
            on_step(t, trk)
    return out


def test_tracker_verification_changes_nothing_else(est, video):
    e, _ = est
    plain = _run(e.tracker(3), video, PLAN)
    checked = _run(e.tracker(3, verify_every=3), video, PLAN)
    for t, (a, b) in enumerate(zip(plain, checked)):
        _same(_without_verify(b), a, f'step {t}')
        assert ('verify' in b[2]) == (t in (3, 6, 9)), t
        if 'verify' in b[2]:
            seqs = range(3) if PLAN[t][0] is None else PLAN[t][0]
            want = e.verify_poses([video[t][s][0] for s in seqs], [video[t][s][1] for s in seqs], b[0])
            _same(b[2]['verify'], want, f'verify {t}')


def test_verifying_step_is_one_graph_and_one_read(est, video):
    from gen6d_b200.graphs import CapturedStage
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    trk = e.tracker(3, verify_every=1, draw='raw')
    plain = e.tracker(3, draw='raw')
    calls = []
    orig = CapturedStage.__call__

    def counted(self, *a):
        calls.append(self)
        return orig(self, *a)
    CapturedStage.__call__ = counted
    try:
        for t in range(3):
            imgs, Ks = [v[0] for v in video[t]], [v[1] for v in video[t]]
            a = plain.step(imgs, Ks)
            drawn_a = {k: [d.cpu().numpy() for d in v] for k, v in a[2]['drawn'].items()}
            calls.clear()
            d0 = IO_BYTES['d2h']
            b = trk.step(imgs, Ks)
            assert len(calls) == 1 and IO_BYTES['d2h'] - d0 == calls[0].static_out[0].numel()
            assert ('verify' in b[2]) == (t > 0)
            _same({k: [d.cpu().numpy() for d in v] for k, v in b[2]['drawn'].items()}, drawn_a, f'drawn {t}')
    finally:
        CapturedStage.__call__ = orig


def test_lost_score_inf_resets_every_sequence(est, video):
    e, _ = est
    a, b = e.tracker(3, verify_every=2, lost_score=np.inf), e.tracker(3)
    plan = [(None, None)] * 6
    got = _run(a, video, plan, lambda t, trk: t != 2 or _check_pending(trk, [True] * 3))
    want = _run(b, video, plan, lambda t, trk: t != 2 or trk.reset())
    for t, (g, w) in enumerate(zip(got, want)):
        _same(_without_verify(g), w, f'step {t}')
    assert got[2][2]['verify']['lost'].all()


def _check_pending(trk, want):
    assert trk._pending.tolist() == want


def test_threshold_at_the_median_resets_the_rows_below(est, video):
    e, _ = est
    probe = _run(e.tracker(3, verify_every=2), video, PLAN[:3])
    scores = probe[2][2]['verify']['score']
    thr = float(np.sort(scores)[1])
    below = [int(s) for s in np.flatnonzero(scores < thr)]
    got = _run(e.tracker(3, verify_every=2, lost_score=thr), video, PLAN[:6])
    want = _run(e.tracker(3), video, PLAN[:6], lambda t, trk: t != 2 or (below and trk.reset(below)))
    for t, (g, w) in enumerate(zip(got, want)):
        _same(_without_verify(g), w, f'step {t}')
    assert got[2][2]['verify']['lost'].tolist() == [s in below for s in range(3)]


# ------------------------------------------------------------------------------------------ objects
@pytest.fixture(scope='module')
def objs(est):
    from gen6d_b200.synthetic import build_estimator, synthetic_database
    e, db = est
    db_b = synthetic_database(seed=8)
    o = e.object_set()
    o.add('a', db)
    o.add('b', db_b)
    return o, {'a': e, 'b': build_estimator(db_b)[0]}


def test_object_set_verify_poses_equals_single_objects(objs, frames, poses):
    o, singles = objs
    imgs, Ks = frames
    p = {'a': poses, 'b': poses[::-1].copy()}
    for thr in [(None, None), (0.0, 0.3)]:
        got = o.verify_poses(imgs, Ks, p, *thr)
        for n, e in singles.items():
            _same(got[n], e.verify_poses(imgs, Ks, p[n], *thr), f'{n} {thr}')


def test_object_tracker_verification(objs, video):
    o, singles = objs
    plain = _run(o.tracker(3), video, PLAN[:7])
    checked = _run(o.tracker(3, verify_every=3), video, PLAN[:7])
    for t, (a, b) in enumerate(zip(plain, checked)):
        for n in o.names:
            _same(_without_verify(b[n]), a[n], f'step {t} {n}')
            assert ('verify' in b[n][2]) == (t in (3, 6))
            if 'verify' in b[n][2]:
                seqs = range(3) if PLAN[t][0] is None else PLAN[t][0]
                want = singles[n].verify_poses([video[t][s][0] for s in seqs], [video[t][s][1] for s in seqs], b[n][0])
                _same(b[n][2]['verify'], want, f'verify {t} {n}')
    # the per-sequence policy: a sequence is re-initialised if any of its objects is lost
    probe = checked[3]
    thr = float(np.median(probe['a'][2]['verify']['score']))
    lost = (probe['a'][2]['verify']['score'] < thr) | (probe['b'][2]['verify']['score'] < thr)
    trk = o.tracker(3, verify_every=3, lost_score=thr)
    _run(trk, video, PLAN[:4])
    assert trk._pending.tolist() == lost.tolist()
