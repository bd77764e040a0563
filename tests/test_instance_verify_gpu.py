"""Verification of the instance trackers (row f21) on the H100: g6d_instances_verify_update against its host twin; a
verifying tracker without thresholds equal to a plain one bit for bit apart from inter['verify'], which appears on exactly
the scheduled steps and equals verify_poses on the same rows; the lost policy with lost_score=+inf and at the median;
staggered and partial steps; every frame form; drawing; one replay and one read per step."""
import cv2
import numpy as np
import pytest
import torch

import instance_verify_oracle as oracle
from gen6d_b200 import frames as fr
from tests.test_instance_track_gpu import two_copy_video
from tests.test_instance_verify_cpu import random_slots, reference, run_twin

pytestmark = pytest.mark.gpu
T = 8                      # frames per video; steps past T replay the video from its start


@pytest.fixture(scope='module')
def db():
    from gen6d_b200.synthetic import synthetic_database
    return synthetic_database(seed=7)


@pytest.fixture(scope='module')
def est(db):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(db)[0]


@pytest.fixture(scope='module')
def videos(db):
    return [two_copy_video(db, T, shift) for shift in (0.0, 15.0, -10.0, 6.0)]


@pytest.fixture(scope='module')
def objs2(est):
    from gen6d_b200.synthetic import synthetic_database
    objs = est.object_set()
    for n, seed in (('a', 7), ('b', 8)):
        objs.add(n, synthetic_database(seed=seed))
    return objs


def _frames(videos, t, seqs):
    return [videos[s][0][t % T] for s in seqs], [videos[s][1] for s in seqs]


def _same(x, y, msg):
    if isinstance(y, dict):
        assert set(x) == set(y), (msg, sorted(x), sorted(y))
        for k in y:
            _same(x[k], y[k], f'{msg} {k}')
        return
    if isinstance(y, (list, tuple)):
        assert len(x) == len(y), msg
        for i, (a, b) in enumerate(zip(x, y)):
            _same(a, b, f'{msg}[{i}]')
        return
    if isinstance(y, torch.Tensor):
        x, y = x.cpu().numpy(), y.cpu().numpy()
    x, y = np.asarray(x), np.asarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, (msg, x.dtype, y.dtype, x.shape, y.shape)
    assert x.tobytes() == y.tobytes(), msg


def _plain(res):
    """A step's result without inter['verify']."""
    return (*res[:3], {k: v for k, v in res[3].items() if k != 'verify'})


def _steps(trk, videos, plan, on_step=None):
    """plan: per step the sequences stepped (None: all).  Returns each step's result (a dict per object for object sets)."""
    out = []
    for t, seqs in enumerate(plan):
        rows = range(trk.S) if seqs is None else seqs
        out.append(trk.step(*_frames(videos, t, rows), sequences=seqs))
        if on_step:
            on_step(t, trk)
    return out


def _per_object(res):
    return res if isinstance(res, dict) else {'': res}


def _state(trk):
    return {k: trk._state[k].cpu().numpy().copy() for k in ('live', 'ids', 'misses')}


# ------------------------------------------------------------------------------------------ 1. kernel == host twin
def test_kernel_equals_host_twin():
    from gen6d_b200 import ops
    rng = np.random.RandomState(5)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for trial in range(60):
        n = int(rng.choice([1, 5, 24, 130, 1000]))
        mm = int(rng.randint(0, 4))
        live, ids, misses = random_slots(rng, n, mm, rng.choice([0.3, 1.0]))
        lost, verified = (rng.rand(n) < 0.5).astype(np.int32), (rng.rand(n) < 0.8).astype(np.int32)
        want = run_twin(lost, verified, mm, live, ids, misses)
        lv, iv, ms = dev(live), dev(ids), dev(misses)
        dropped = ops.instances_verify_update(dev(lost), dev(verified), mm, lv, iv, ms)
        for g, w, k in zip((lv, iv, ms, dropped), want, ('live', 'ids', 'misses', 'dropped')):
            _same(g.cpu().numpy(), w, f'{trial} {k}')
        _same(want, oracle.verify_update(lost, verified, mm, live, ids, misses), f'{trial} oracle')


# ------------------------------------------------------------------------------------------ 2. thresholds None change nothing
def _check_rows(verify_poses, res, frames_of, Ks_of, M, S, det_seqs, msg):
    """inter['verify'] of a step equals verify_poses on the same rows (slot m of sequence s, m-major: the tracker's batch
    order) with the step's float32 poses, on the live slots of the sequences that did not re-detect (det_seqs)."""
    for name, (poses, _, ids, inter) in _per_object(res).items():
        rows = [(s, m) for m in range(M) for s in range(S)]
        want = verify_poses(name, [frames_of[s] for s, _ in rows], [Ks_of[s] for s, _ in rows],
                            np.stack([poses[s, m] for s, m in rows]))
        live = [ids[s, m] >= 0 and s not in det_seqs for s, m in rows]
        assert any(live), msg
        for k, w in want.items():
            g = np.stack([inter['verify'][k][s, m] for s, m in rows])
            _same(g[live], w[live], f'{msg} {name} {k}')


def _verify_poses_of(trk):
    if hasattr(trk, 'objs'):
        return lambda name, f, K, p: trk.objs.verify_poses(f, K, {n: p for n in trk.names})[name]
    return lambda name, f, K, p: trk.est.verify_poses(f, K, p)


@pytest.mark.parametrize('case', ['lockstep', 'per_sequence', 'staggered', 'objects'])
def test_thresholds_none_change_nothing(est, objs2, videos, case):
    S, M = 3, 2
    steps = 30 if case == 'lockstep' else 14
    if case == 'objects':
        make = lambda **kw: objs2.instance_tracker(S, max_instances=M, redetect_every=6, **kw)
        every = 4
    else:
        sch = case
        make = lambda **kw: est.instance_tracker(S, max_instances=M, redetect_every=7 if sch == 'lockstep' else 4, schedule=sch, **kw)
        every = {'lockstep': 3, 'per_sequence': 2, 'staggered': 2}[case]
    plan = [None] * steps
    if case == 'per_sequence':
        plan = [None, None, [2, 0], [1], None, [0, 1], None, [2], None, None, [1, 2], None, [0], None]
    plain, checked = make(), make(verify_every=every)
    a, b = _steps(plain, videos, plan), _steps(checked, videos, plan)
    # the steps that should verify, from the sequences each step stepped and re-detected
    sched = []
    for t, seqs in enumerate(plan):
        r = next(iter(_per_object(a[t]).values()))
        stepped = list(range(S)) if seqs is None else list(seqs)
        det = r[3].get('detected')                   # in the step's sequence order
        if det is None:
            det_seqs = set(stepped) if 'det_slot' in r[3] else set()
        else:
            det_seqs = {s for s, d in zip(stepped, det) if d}
        sched.append((stepped, det_seqs))
    want_steps = reference(S, every, sched)
    assert want_steps, case
    vp = _verify_poses_of(checked)
    for t in range(steps):
        for name in _per_object(a[t]):
            _same(_plain(_per_object(b[t])[name]), _per_object(a[t])[name], f'{case} step {t} {name}')
            assert ('verify' in _per_object(b[t])[name][3]) == (t in want_steps), (case, t)
        if t in want_steps and plan[t] is None:
            _check_rows(vp, b[t], *_frames(videos, t, range(S)), M, S, sched[t][1], f'{case} step {t}')


# ------------------------------------------------------------------------------------------ 3. the lost policy
def test_lost_score_inf_drops_or_keeps(est, videos):
    S, M = 2, 2
    for mm in (0, 1):
        trk = est.instance_tracker(S, max_instances=M, max_misses=mm, verify_every=2, lost_score=np.inf)
        res = _steps(trk, videos, [None] * 4)
        ids2, v = res[2][2], res[2][3]['verify']
        live_ids = sorted(int(i) for i in ids2.reshape(-1) if i >= 0)
        assert live_ids and v['lost'][ids2 >= 0].all()
        assert 'det_slot' not in res[2][3] and 'det_slot' in res[3][3]            # the next step re-detects
        after = set(int(i) for i in res[3][2].reshape(-1) if i >= 0)
        if mm == 0:
            assert v['dropped'] == live_ids
            assert not after & set(live_ids) and min(after) > max(live_ids)     # new tracks, new ids
            continue
        assert v['dropped'] == []
        assert after & set(live_ids)                                            # the association keeps matched ids
        # every track holds one miss: the re-detection keeps what it matches and drops the rest, as a plain tracker
        # with max_misses=0 told to redetect() does
        plain = est.instance_tracker(S, max_instances=M, max_misses=0)
        want = _steps(plain, videos, [None] * 4, lambda t, p: t != 2 or p.redetect())
        for t in range(4):
            _same(_plain(res[t]), want[t], f'step {t}')


def test_median_lost_score_misses_exactly_the_rows_below(est, videos):
    S, M = 3, 2
    make = lambda **kw: est.instance_tracker(S, max_instances=M, max_misses=3, schedule='per_sequence', **kw)
    probe = _steps(make(verify_every=2), videos, [None] * 3)[2]
    live = probe[2] >= 0
    thr = float(np.median(probe[3]['verify']['score'][live]))
    trk = make(verify_every=2, lost_score=thr)
    _steps(trk, videos, [None] * 2)
    before = _state(trk)
    res = trk.step(*_frames(videos, 2, range(S)))
    v = res[3]['verify']
    lost = live & ~(v['score'] >= thr)
    assert lost.any() and not lost.all()
    _same(v['lost'], lost, 'lost rows')
    # the slot state follows the host twin; the rows are m-major (row m*S + s)
    n = M * S
    want = run_twin(lost.T.reshape(n).astype(np.int32), np.ones(n, np.int32), 3, before['live'], before['ids'], before['misses'])
    after = _state(trk)
    for k, w in zip(('live', 'ids', 'misses'), want[:3]):
        _same(after[k], w, k)
    assert v['dropped'] == []
    lost_seqs = lost.any(1)
    _same(trk.detecting(), lost_seqs, 'due')
    nxt = trk.step(*_frames(videos, 3, range(S)))
    _same(nxt[3]['detected'], lost_seqs, 'detected next')


def test_staggered_verifies_on_mixed_steps(est, videos):
    S, M = 4, 2
    trk = est.instance_tracker(S, max_instances=M, redetect_every=3, schedule='staggered', verify_every=1)
    res = _steps(trk, videos, [None] * 6)
    for t in range(1, 6):
        det = res[t][3]['detected']
        assert det.any() and not det.all(), t                               # a mixed step ...
        v = res[t][3]['verify']                                              # ... that verifies
        assert np.isnan(v['score'][det]).all() and not v['lost'][det].any()
        live = (res[t][2] >= 0) & ~det[:, None]
        assert live.any() and np.isfinite(v['window_scale'][live]).all()


# ------------------------------------------------------------------------------------------ 4. frame forms and drawing
def _nv12(img):
    h, w = img.shape[:2]
    i420 = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    yuv = np.vstack([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])
    surf = torch.from_numpy(yuv).cuda()
    return fr.NV12(surf[:h], surf[h:]), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)


@pytest.mark.parametrize('form', ['cuda', 'nv12', 'resized', 'two_sizes'])
def test_frame_forms_equal_numpy(est, videos, form):
    S, M = 2, 2
    make = lambda: est.instance_tracker(S, max_instances=M, verify_every=1, lost_score=0.0)
    dev_trk, ref_trk = make(), make()
    for t in range(3):
        imgs, Ks = _frames(videos, t, range(S))
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
        else:
            ref = [i if j % 2 else np.ascontiguousarray(i[16:464, 32:608]) for j, i in enumerate(imgs)]
            Ks = [K if j % 2 else K - np.asarray([[0, 0, 32], [0, 0, 16], [0, 0, 0]]) for j, K in enumerate(Ks)]
            dev = [torch.from_numpy(i).cuda() for i in ref]
        got, want = dev_trk.step(dev, Ks), ref_trk.step(ref, Ks)
        _same(got, want, f'{form} step {t}')
        assert ('verify' in got[3]) == (t > 0)


def test_drawing_is_unchanged(est, videos):
    S, M = 2, 2
    make = lambda **kw: est.instance_tracker(S, max_instances=M, draw='raw', **kw)
    plain, checked = make(), make(verify_every=1)
    for t in range(5):
        imgs, Ks = _frames(videos, t, range(S))
        if t < 3:                                    # tracker-owned frames
            a, b = plain.step(imgs, Ks), checked.step(imgs, Ks)
            drawn = lambda r: {k: [d.cpu() for d in v] for k, v in r[3]['drawn'].items()}
            _same(drawn(b), drawn(a), f'drawn {t}')
        else:                                        # the caller's destinations
            out_a = {'raw': [torch.zeros(i.shape, dtype=torch.uint8, device='cuda') for i in imgs]}
            out_b = {'raw': [torch.zeros(i.shape, dtype=torch.uint8, device='cuda') for i in imgs]}
            a, b = plain.step(imgs, Ks, out=out_a), checked.step(imgs, Ks, out=out_b)
            _same(out_b['raw'], out_a['raw'], f'out= {t}')
        assert ('verify' in b[3]) == (t > 0)
        _same(_plain(b), a, f'step {t}')


def test_one_replay_and_one_read_per_step(est, videos):
    from gen6d_b200.graphs import CapturedStage
    from gen6d_b200.network.base import IO_BYTES
    S, M = 3, 2
    trk = est.instance_tracker(S, max_instances=M, redetect_every=3, schedule='staggered', verify_every=1, lost_score=0.0)
    calls = []
    orig = CapturedStage.__call__

    def counted(self, *a):
        calls.append(self)
        return orig(self, *a)
    CapturedStage.__call__ = counted
    try:
        for t in range(5):
            calls.clear()
            d0 = IO_BYTES['d2h']
            res = trk.step(*_frames(videos, t, range(S)))
            assert len(calls) == 1 and IO_BYTES['d2h'] - d0 == calls[0].static_out[0].numel(), t
            assert ('verify' in res[3]) == (t > 0)
    finally:
        CapturedStage.__call__ = orig
    print('graph kernels', {key[0]: s.kernels for key, s in trk.stages.stages.items()})
