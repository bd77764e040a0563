"""Per-sequence re-detection of the instance trackers (row f18) on the H100: g6d_instances_associate_sequences against its
host twin, 'per_sequence' stepped in lockstep against 'lockstep' bit for bit, the mixed instance step (one sequence
re-detecting while the others refine) against predict_instances and a lockstep refine step, partial steps against
single-sequence trackers, and one replay and one read per step with one graph per (b, d)."""
import numpy as np
import pytest
import torch

from tests.test_instance_track_gpu import DET_KEYS, SENS, _frames, _pose_bound, two_copy_video

pytestmark = pytest.mark.gpu
REFINE_BAR = 2e-4          # test_track_partial_gpu.py's lockstep bar: one refinement at another batch size
FULL_BAR = max(2.0 * float(SENS['gain_R'][-1]) * 1e-3, 2e-3)      # test_instances_gpu.py's bar after a full chain


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
    return [two_copy_video(db, 8, shift) for shift in (0.0, 15.0, -10.0, 6.0)]


@pytest.fixture(scope='module')
def objs2(est):
    from gen6d_b200.synthetic import synthetic_database
    objs = est.object_set()
    for n, seed in (('a', 7), ('b', 8)):
        objs.add(n, synthetic_database(seed=seed))
    return objs


def _same(x, y, msg):
    x, y = np.asarray(x), np.asarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, (msg, x.dtype, y.dtype, x.shape, y.shape)
    assert x.tobytes() == y.tobytes(), msg


def _same_result(got, want, msg, skip=('detected',)):
    for a, b, k in zip(got[:3], want[:3], ('poses', 'smoothed', 'ids')):
        _same(a, b, f'{msg} {k}')
    gi, wi = got[3], want[3]
    assert set(gi) - set(skip) == set(wi) - set(skip), (msg, sorted(gi), sorted(wi))
    for k in wi:
        if k in skip:
            continue
        if k == 'refine_poses':
            assert len(gi[k]) == len(wi[k]), msg
            for i, (a, b) in enumerate(zip(gi[k], wi[k])):
                _same(a, b, f'{msg} refine_poses[{i}]')
        elif k == 'dropped':
            assert gi[k] == wi[k], msg
        else:
            _same(gi[k], wi[k], f'{msg} {k}')


def _state(trk):
    return {k: v.cpu().numpy().copy() for k, v in trk._state.items()} | {'next_id': trk._next_id.cpu().numpy().copy()}


# ------------------------------------------------------------------------------------------ 1. kernel == host twin
def test_kernel_equals_host_twin():
    from gen6d_b200 import ops
    from gen6d_b200.instance_track import host_associate_sequences
    from tests.test_instance_track_cpu import OUTS, STATE
    from tests.test_instance_track_schedule_cpu import random_case
    rng = np.random.RandomState(17)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    for trial in range(150):
        p, det_index, batch, K, S, M, D = random_case(rng, int(rng.choice([1, 2])))
        q = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
        want = host_associate_sequences(det_index, batch['det'], batch['valid'], batch['init'], q['cams'], q['centers'], q['res'],
                                        q['gate'], q['max_misses'], q['F'], q['r'], q['prev'], *[q[k] for k in STATE])
        st = {k: dev(p[k]) for k in STATE}
        got = ops.instances_associate_sequences(dev(det_index.astype(np.int32)), dev(batch['det']), dev(batch['valid']),
                                                dev(batch['init']), dev(p['cams']), dev(p['centers']), p['res'], p['gate'],
                                                p['max_misses'], p['F'], p['r'], dev(p['prev']), *[st[k] for k in STATE])
        for k, g, w in zip(OUTS, got, want):
            _same(g.cpu().numpy(), w, f'{trial} {k}')
        for k in STATE:
            _same(st[k].cpu().numpy(), q[k], f'{trial} {k}')
    from tests.test_objects_instance_track_cpu import make_set_problem
    p, K, S, M = make_set_problem(np.random.RandomState(1), 1, S=2, M=2, F=2, r=1)
    st = {k: dev(p[k]) for k in STATE}
    with pytest.raises(ValueError, match='twice'):
        ops.instances_associate_sequences(dev(np.zeros(S, np.int32)), dev(np.zeros((M, 4), np.float32)), dev(np.zeros(M, np.int32)),
                                          dev(np.zeros((M, 12))), dev(p['cams']), dev(p['centers']), p['res'], p['gate'],
                                          p['max_misses'], p['F'], p['r'], dev(p['prev']), *[st[k] for k in STATE])


# ------------------------------------------------------------------------------------------ 2. per_sequence in lockstep
def _lockstep_equivalence(make, step, videos, S):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    a, b = make('lockstep'), make('per_sequence')
    for t in range(6):
        if t == 4:
            a.reset()
            b.reset()
        imgs, Ks = _frames(videos, t, S)
        k0 = REPLAYED_KERNELS[0]
        want = step(a, imgs, Ks)
        k1 = REPLAYED_KERNELS[0]
        got = step(b, imgs, Ks)
        assert REPLAYED_KERNELS[0] - k1 == k1 - k0, t
        for name in want:
            _same_result(got[name], want[name], f'step {t} {name}')
            assert got[name][3]['detected'].all() == ('spawned' in want[name][3]), t
        for k, v in _state(a).items():
            _same(_state(b)[k], v, f'step {t} state {k}')
    assert len(b.stages.stages) == len(a.stages.stages)


def test_per_sequence_in_lockstep_equals_lockstep(est, videos):
    S = 3
    _lockstep_equivalence(lambda sch: est.instance_tracker(num_sequences=S, max_instances=2, redetect_every=2, schedule=sch),
                          lambda trk, imgs, Ks: {'': trk.step(imgs, Ks)}, videos, S)


def test_per_sequence_in_lockstep_equals_lockstep_objects(objs2, videos):
    S = 2
    _lockstep_equivalence(lambda sch: objs2.instance_tracker(num_sequences=S, max_instances=2, redetect_every=2, schedule=sch),
                          lambda trk, imgs, Ks: trk.step(imgs, Ks), videos, S)


# ------------------------------------------------------------------------------------------ 3. the mixed step
def test_mixed_step(est, videos):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.instance_track import host_associate_sequences
    from gen6d_b200.network.base import IO_BYTES
    S, M = 3, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, schedule='per_sequence')
    ref = est.instance_tracker(num_sequences=S, max_instances=M)
    for t in range(2):
        imgs, Ks = _frames(videos, t, S)
        trk.step(imgs, Ks)
        ref.step(imgs, Ks)
    before = _state(trk)
    trk.reset([1])
    assert trk.detecting().tolist() == [False, True, False]
    imgs, Ks = _frames(videos, 2, S)
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    p, sm, ids, inter = trk.step(imgs, Ks)
    stage = [st for key, st in trk.stages.stages.items() if key[0][0] == 'instance_mixed']
    assert len(stage) == 1 and REPLAYED_KERNELS[0] - k0 == stage[0].kernels
    assert IO_BYTES['d2h'] - d0 == stage[0].static_out[0].numel()
    assert inter['detected'].tolist() == [False, True, False]
    # sequence 1: predict_instances on its frame
    wp, want = est.predict_instances([imgs[1]], [Ks[1]], max_instances=M)
    for k in DET_KEYS + ('instance_valid',):
        _same(inter[k][1:2], want[k], k)
    for k in ('det_position', 'det_score', 'sel_scores'):
        assert np.isnan(inter[k][[0, 2]]).all(), k
    assert (inter['sel_ref_idx'][[0, 2]] == -1).all() and not inter['instance_valid'][[0, 2]].any()
    assert (inter['det_slot'][[0, 2]] == -1).all() and not inter['spawned'][[0, 2]].any()
    # sequences 0 and 2: a lockstep refine step from the same state
    rp, rsm, rids, rinter = ref.step(imgs, Ks)
    for s in (0, 2):
        _same(ids[s], before['ids'].reshape(M, S)[:, s], f'ids {s}')
        _same(ids[s], rids[s], f'ids {s}')
        _same(p[s], rp[s], f'poses {s}')
        _same(sm[s], rsm[s], f'smoothed {s}')
        _same(inter['refine_poses'][0][s].astype(np.float32), rinter['refine_poses'][0][s], f'chain 0 {s}')
        for i in range(1, len(inter['refine_poses'])):                  # a shorter chain repeats its final pose
            _same(inter['refine_poses'][i][s], rinter['refine_poses'][min(i, trk.refine_iter)][s], f'chain {i} {s}')
    # sequence 1's refinement (one stage over all rows, then two over the re-detecting slots) against predict_instances'
    valid = want['instance_valid'][0]
    assert valid[0] and (inter['det_slot'][1][valid] == np.arange(M)[valid]).all()
    _pose_bound([c[1][valid] for c in inter['refine_poses']], [c[0][valid] for c in want['refine_poses']], 'mixed seq 1')
    assert np.abs(p[1][valid].astype(np.float64) - wp[0][valid]).max() <= FULL_BAR
    # the association state: the host twin fed this step's own detections
    after = _state(trk)
    q = {k: v.copy() for k, v in before.items()}
    q['live'][np.arange(M) * S + 1] = 0
    q['ids'][np.arange(M) * S + 1] = -1
    q['misses'][np.arange(M) * S + 1] = 0
    q['ring'][np.arange(M) * S + 1] = 0
    q['count'][np.arange(M) * S + 1] = 0
    det = np.concatenate([inter['det_position'][1], inter['det_scale_r2q'][1][:, None], inter['det_score'][1][:, None]], 1)
    from gen6d_b200 import glue
    cams = glue.cameras(np.stack(Ks))
    init = np.ascontiguousarray(np.asarray(want['refine_poses'][0][0], np.float64).reshape(M, 12))
    _, _, lists, det_slot, spawned, dropped = host_associate_sequences(np.array([-1, 0, -1]), det.astype(np.float32), inter['instance_valid'][1].astype(np.int32), init,
                             cams, np.asarray(est.ref_info['center'], np.float64).reshape(1, 3), est.cfg['ref_resolution'],
                             trk.gate, trk.max_misses, est.cfg['refine_iter'], trk.refine_iter, before['prev'], q['live'], q['ids'],
                             q['misses'], q['next_id'], q['park'], q['ring'], q['count'])
    for k in ('live', 'ids', 'misses', 'next_id'):
        _same(after[k], q[k], k)
    fin = np.isfinite(q['park']).all(1)
    _same(after['park'][fin], q['park'][fin], 'park')
    assert fin.reshape(M, S)[:, [0, 2]].all()
    _same(inter['det_slot'][1], det_slot.reshape(M, S)[:, 1].astype(np.int64), 'det_slot')
    _same(inter['spawned'][1], spawned.reshape(M, S)[:, 1].astype(bool), 'spawned')
    assert inter['dropped'] == sorted(int(i) for i in dropped if i >= 0)
    F = est.cfg['refine_iter']
    assert len(lists) == M * S * trk.refine_iter + M * 1 * (F - trk.refine_iter)      # one stage over all rows


# ------------------------------------------------------------------------------------------ 4. partial steps
def test_partial_steps_equal_single_sequence_trackers(est, videos):
    """S = 4 staggered (E = 3), seeded subsets with a reset([2]) and a redetect([0]) mid-run.  Every step: which streams
    re-detect follows the staggered rule stated here per stream; each listed stream equals a num_sequences=1 tracker
    started from that stream's state rows and fed its frame and its re-detection -- live slots, kept ids, spawns, drops
    and det_slot exactly, poses within REFINE_BAR on refine-only rows and FULL_BAR after a re-detection (the stream's
    detection, selection and refinement ran at another batch size); ids are unique tracker-wide and idle sequences keep
    their state bytes."""
    S, M, E = 4, 2, 3
    trk = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=E, schedule='staggered')
    ref = est.instance_tracker(num_sequences=1, max_instances=M, schedule='per_sequence')
    rng = np.random.RandomState(4)
    t_of = [0] * S
    pend, cnt = np.ones(S, bool), np.zeros(S, int)              # the expected schedule, per stream
    worst = {True: 0.0, False: 0.0}
    for step in range(10):
        if step == 4:
            trk.reset([2])
            pend[2] = True
        if step == 6:
            trk.redetect([0])
            pend[0] = True
        seqs = [int(s) for s in rng.permutation(S)[:rng.randint(1, S + 1)] if t_of[s] < 8]
        if not seqs:
            continue
        due = pend | (cnt >= E)
        before = _state(trk)
        imgs = [videos[s][0][t_of[s]] for s in seqs]
        Ks = [videos[s][1] for s in seqs]
        p, sm, ids, inter = trk.step(imgs, Ks, sequences=seqs)
        assert inter['sequences'].tolist() == seqs
        assert inter['detected'].tolist() == due[seqs].tolist(), (step, seqs)
        after = _state(trk)
        for s in range(S):
            rows = np.arange(M) * S + s
            if s not in seqs:
                for k in ('prev', 'park', 'live', 'ids', 'misses', 'ring', 'count'):
                    _same(after[k][rows], before[k][rows], f'{step} idle {s} {k}')
        for i, s in enumerate(seqs):
            rows = np.arange(M) * S + s
            for k in ('prev', 'park', 'live', 'ids', 'misses', 'ring', 'count'):
                ref._state[k].copy_(torch.from_numpy(before[k][rows]).cuda())
            ref._next_id.copy_(torch.from_numpy(before['next_id']).cuda())
            ref._schedule.pending[:] = due[s]
            rp, rsm, rids, rinter = ref.step([imgs[i]], [Ks[i]])
            assert rinter['detected'][0] == due[s]
            assert ((ids[i] >= 0) == (rids[0] >= 0)).all(), (step, s)
            if due[s]:
                for k in ('det_slot', 'spawned'):
                    _same(inter[k][i], rinter[k][0], f'{step} {k} {s}')
                kept = (ids[i] >= 0) & ~inter['spawned'][i]
            else:
                kept = ids[i] >= 0
            _same(ids[i][kept], rids[0][kept], f'{step} ids {s}')
            ok = ids[i] >= 0
            if ok.any():
                d = float(np.abs(p[i][ok].astype(np.float64) - rp[0][ok]).max())
                worst[bool(due[s])] = max(worst[bool(due[s])], d)
                assert d <= (FULL_BAR if due[s] else REFINE_BAR), (step, s, d)
            t_of[s] += 1
        live_ids = after['ids'][after['ids'] >= 0]
        assert len(np.unique(live_ids)) == len(live_ids), step
        # the expected counters: a detection leaves 1, a marked one 1 + floor(s*E/S); idle streams keep theirs
        for s in seqs:
            cnt[s] = (1 + s * E // S if pend[s] else 1) if due[s] else cnt[s] + 1
            pend[s] = False
    print('partial steps vs single-sequence trackers, max |dpose| (re-detecting, refining)', worst[True], worst[False])


# ------------------------------------------------------------------------------------------ 5. padding canary
def test_padding_detection_row_changes_no_real_row(est, videos, monkeypatch):
    """A mixed step of S = 4 with sequences 0, 1 and 3 re-detecting (detection batch d = 4, padding row 3): pointing the
    padding row at sequence 2's frame instead of a copy of sequence 3's changes no state byte and no real row of the
    results.  The refiner stages list M*S rows once, then M*d rows."""
    from gen6d_b200 import glue, ops
    from gen6d_b200.instance_track import plan_mixed
    S, M = 4, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, schedule='per_sequence')
    imgs, Ks = _frames(videos, 0, S)
    trk.step(imgs, Ks)
    imgs, Ks = _frames(videos, 1, S)
    det_seq = np.array([True, True, False, True])
    seq, _, det_index, d, _ = plan_mixed(det_seq, None)
    assert seq.tolist() == [0, 1, 3, 3] and d == 4
    sizes = []
    orig = ops.glue_refine_problems_rows
    monkeypatch.setattr(ops, 'glue_refine_problems_rows', lambda *a: sizes.append(a[6].shape[0]) or orig(*a))
    fn = trk._body(trk._tables(), 'mixed', S, d)
    frames = torch.from_numpy(np.stack(imgs)).cuda()
    cams = est.detector._to_dev(glue.cameras(np.stack(Ks)))
    x = trk._state
    outs = []
    with torch.no_grad():
        for last in (3, 2):
            state = [x['prev'], x['park'], x['live'], x['ids'], x['misses'], trk._next_id, x['ring'], x['count']]
            state = [t.clone() for t in state]
            pad = torch.from_numpy(np.array([0, 1, 3, last], np.int64)).cuda()
            o = fn(frames, cams, *state, pad, torch.from_numpy(det_index.astype(np.int32)).cuda())
            outs.append([t.cpu().numpy().copy() for t in o])
    G, n, F, r = M, M * S, est.cfg['refine_iter'], trk.refine_iter
    assert sizes == [G * S] * r + [G * d] * (F - r) + [G * S] * r + [G * d] * (F - r), sizes
    for k, (a, b) in enumerate(zip(outs[0][1:], outs[1][1:])):
        _same(b, a, f'state output {k}')
    n_chain = max(F, r) + 1
    head = (n_chain * n * 12 + n * 12 + n * 16 + n * trk.num * 16 + n + n) * 8      # chain, smoothed, avg, ring, count, ids
    _same(outs[1][0][:head], outs[0][0][:head], 'packed results')
    res = [trk._decode(o[0], True, S, det_index, d)[0] for o in outs]
    for k in DET_KEYS + ('instance_valid', 'det_slot', 'spawned'):
        _same(res[1][3][k], res[0][3][k], k)


# ------------------------------------------------------------------------------------------ 6. inputs and drawing
SCHED = [[0, 2, 3], [1, 2], [3, 0], [2], [0, 1, 2, 3], [1, 3, 0]]


def _kind_inputs(kind, imgs, seqs):
    from tests.test_track_partial_gpu import _inputs, _two_sizes
    if kind == 'two_sizes':
        imgs = _two_sizes(imgs, seqs)
        return [torch.from_numpy(im).cuda() for im in imgs], imgs
    return _inputs(kind, imgs)


@pytest.mark.parametrize('kind', ['cuda', 'nv12', 'resized', 'two_sizes'])
def test_frame_kinds_equal_the_numpy_path(est, videos, kind):
    """Mixed and partial steps (SCHED with a reset([1]) and a redetect([3]) between) on device frames equal the numpy path
    on the frames the graph holds, every result byte."""
    S, M = 4, 2
    a, b = [est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=3, schedule='staggered') for _ in range(2)]
    kinds = set()
    for t, seqs in enumerate(SCHED):
        if t == 2:
            a.reset([1]), b.reset([1])
        if t == 4:
            a.redetect([3]), b.redetect([3])
        imgs = [np.ascontiguousarray(videos[s][0][t]) for s in seqs]
        ins, ref = _kind_inputs(kind, imgs, seqs)
        Ks = [videos[s][1] for s in seqs]
        kinds.add(tuple(a.detecting()[seqs]))
        got, want = a.step(ins, Ks, sequences=seqs), b.step(ref, Ks, sequences=seqs)
        _same_result(got, want, f'{kind} step {t}', skip=())
    assert any(0 < sum(k) < len(k) for k in kinds), kinds                 # some step was mixed


def test_drawing_and_destinations(est, videos):
    """draw='smoothed' in mixed and partial steps: every live slot drawn as cv2's draw_bbox_3d with the step's own smoothed
    poses, results equal a non-drawing tracker's, out= buffers of idle sequences keep their bytes."""
    from tests.test_draw_cpu import cv_draw_bbox_3d, project
    S, M = 4, 2
    dt = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=3, schedule='staggered', draw='smoothed')
    nt = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=3, schedule='staggered')

    def expect(img, sm, ids, K):
        for m in range(M):
            if ids[m] >= 0:
                img = cv_draw_bbox_3d(img, project(dt.bbox, sm[m], K), (0, 0, 255))
        return img
    n_live = 0
    for t, seqs in enumerate(SCHED + [[3, 0], [2], [1, 3, 0]]):
        if t == 2:
            dt.reset([1]), nt.reset([1])
        imgs = [np.ascontiguousarray(videos[s][0][t % 8]) for s in seqs]
        Ks = [videos[s][1].astype(np.float32) for s in seqs]
        if t < len(SCHED):
            p, sm, ids, inter = dt.step(imgs, Ks, sequences=seqs)
            drawn = inter.pop('drawn')['smoothed']
        else:
            h, w = imgs[0].shape[:2]
            bufs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda') for _ in range(S)]
            keep = [x.clone() for x in bufs]
            p, sm, ids, inter = dt.step(imgs, Ks, out={'smoothed': [bufs[s] for s in seqs]}, sequences=seqs)
            assert 'drawn' not in inter
            drawn = [bufs[s] for s in seqs]
            for s in range(S):
                if s not in seqs:
                    assert torch.equal(bufs[s], keep[s]), (t, s)
        _same_result((p, sm, ids, inter), nt.step(imgs, Ks, sequences=seqs), f'step {t}', skip=())
        assert len(drawn) == len(seqs)
        for i in range(len(seqs)):
            n_live += int((ids[i] >= 0).sum())
            np.testing.assert_array_equal(drawn[i].cpu().numpy(), expect(imgs[i], sm[i], ids[i], Ks[i]), err_msg=f'{t} {i}')
    assert n_live > 0


# ------------------------------------------------------------------------------------------ 7. one replay, one read
def test_one_replay_one_read_per_step(est, videos):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    S = 4
    trk = est.instance_tracker(num_sequences=S, max_instances=2, redetect_every=2, schedule='staggered')
    for t in range(5):
        imgs, Ks = _frames(videos, t, S)
        k0, d0, n0 = REPLAYED_KERNELS[0], IO_BYTES['d2h'], len(trk.stages.stages)
        trk.step(imgs, Ks)
        dk = REPLAYED_KERNELS[0] - k0
        assert dk in [st.kernels for st in trk.stages.stages.values()], t
        assert IO_BYTES['d2h'] - d0 in [st.static_out[0].numel() for st in trk.stages.stages.values()], t
        assert len(trk.stages.stages) - n0 <= 1


def test_errors(est):
    trk = est.instance_tracker(num_sequences=2, max_instances=2)
    with pytest.raises(ValueError, match='sequences='):
        trk.step([np.zeros((48, 64, 3), np.uint8)], [np.eye(3)], sequences=[0])
    with pytest.raises(ValueError, match='lockstep'):
        trk.redetect([0])
    with pytest.raises(ValueError, match='redetect_every'):
        est.instance_tracker(num_sequences=2, schedule='staggered')
    with pytest.raises(ValueError, match='schedule'):
        est.instance_tracker(num_sequences=2, schedule='sometimes')
