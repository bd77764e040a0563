"""Boxes from another detector (row f19) on the H100: g6d_det_from_boxes against its host twin, predict_instances /
predict_batch / ObjectSet.predict_instances with boxes against the same calls whose detection step returns the host
twin's records, frame kinds, CUDA boxes, the graph without the detector's kernels, a round trip through the detector's
own records, and the instance trackers' box steps (lockstep and per sequence)."""
import numpy as np
import pytest
import torch

import boxes_oracle as O
from gen6d_b200 import boxes as B
from gen6d_b200 import ops
from tests.test_instance_track_gpu import DET_KEYS, _frames, two_copy_video
from tests.test_track_partial_gpu import _inputs, _two_sizes

pytestmark = pytest.mark.gpu
INV = B.inv_box_size(128)
KEYS = DET_KEYS + ('instance_valid', 'instance_count')


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
    return [two_copy_video(db, 6, shift) for shift in (0.0, 15.0, -10.0)]


@pytest.fixture(scope='module')
def found(est, videos):
    """The detector's own instances on the first frame of each video, as boxes (squares of side 128 * scale)."""
    imgs, Ks = _frames(videos, 0, 3)
    _, inter = est.predict_instances(imgs, Ks, max_instances=2)
    return imgs, Ks, [_boxes_of(inter, f) for f in range(3)], inter


def _boxes_of(inter, f):
    keep = inter['instance_valid'][f]
    (x, y), s, sc = inter['det_position'][f, keep].T, inter['det_scale_r2q'][f, keep], inter['det_score'][f, keep]
    half = 64.0 * s
    return np.stack([x - half, y - half, x + half, y + half, sc], 1).astype(np.float32)


def _same(x, y, msg):
    x, y = np.asarray(x), np.asarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, (msg, x.dtype, y.dtype, x.shape, y.shape)
    assert x.tobytes() == y.tobytes(), msg


def _same_inter(got, want, msg):
    assert set(got) == set(want), (msg, sorted(got), sorted(want))
    for k in want:
        if k == 'refine_poses':
            assert len(got[k]) == len(want[k])
            for i, (a, b) in enumerate(zip(got[k], want[k])):
                _same(a, b, f'{msg} refine_poses[{i}]')
        elif k == 'dropped':
            assert got[k] == want[k], msg
        elif k != 'drawn':
            _same(got[k], want[k], f'{msg} {k}')


def _twin_detection(monkeypatch, target, table, M):
    """Replace target._peaks_detect_fn by a detection step that returns the host twin's records of `table` (uploaded
    now, outside any capture)."""
    det, valid, count = B.host_records(table[0], table[1], M, INV)
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (('det', det), ('valid', valid), ('count', count))}

    def fake(*key):
        extra = []

        def detect(frames):
            extra[:] = [d['valid'].reshape(-1), d['count']]
            return d['det'].reshape(-1, 4)
        return detect, extra
    monkeypatch.setattr(target, '_peaks_detect_fn', fake)


def _host_table(t):
    buf = t.host()
    n = t.n_maps * t.N * 5
    return buf[:n].reshape(t.n_maps, t.N, 5), buf[n:].view(np.int32)


# ------------------------------------------------------------------------------------------ the kernel
def test_kernel_equals_host_twin():
    rng = np.random.RandomState(3)
    for N in (1, 2, 16, 256):
        for M in (1, 4, 16):
            t, c = O.random_table(rng, 13, N)
            det, valid, count = ops.det_from_boxes(torch.from_numpy(t).cuda(), torch.from_numpy(c).cuda(), M, INV)
            for g, w, k in zip((det, valid, count), B.host_records(t, c, M, INV), ('det', 'valid', 'count')):
                _same(g.cpu().numpy(), w, f'N={N} M={M} {k}')


# ------------------------------------------------------------------------------------------ predict_instances
@pytest.mark.parametrize('M', [1, 4])
def test_predict_instances_equals_the_twin_detection(est, found, monkeypatch, M):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    imgs, Ks, boxes, _ = found
    boxes = [boxes[0], np.zeros((0, 5), np.float32), np.concatenate([boxes[2], boxes[1][:1] + 3])]
    est.stages.clear()
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    gp, got = est.predict_instances(imgs, Ks, max_instances=M, boxes=boxes)
    (stage,) = est.stages.stages.values()
    N = B.bucket(max(len(b) for b in boxes))
    assert stage.static_in[-1].shape == (3 * N * 5 + 3,)
    assert REPLAYED_KERNELS[0] - k0 == stage.kernels and IO_BYTES['d2h'] - d0 == stage.static_out.numel()
    gp2, got2 = est.predict_instances(imgs, Ks, max_instances=M, boxes=boxes)        # replays
    assert len(est.stages.stages) == 1
    _same(gp2, gp, 'replay')
    box_kernels = stage.kernels
    # the same call with the detector's maps and peaks: its graph minus the detector's kernels, plus the box kernel
    est.stages.clear()
    est.predict_instances(imgs, Ks, max_instances=M)
    (det_stage,) = est.stages.stages.values()
    from gen6d_b200 import _lib
    frames = est.detector.upload_frame(imgs)
    with torch.no_grad():
        detect, _ = est._peaks_detect_fn(M, 1, 0.3, None)
        n0 = _lib.launch_count()
        detect(frames)
        n_det = _lib.launch_count() - n0
    assert box_kernels == det_stage.kernels - n_det + 1, (box_kernels, det_stage.kernels, n_det)
    # against the detection step swapped for the host twin's records
    est.stages.clear()
    _twin_detection(monkeypatch, est, _host_table(B.for_frames(boxes, 3, 'x', 'cuda:0')), M)
    wp, want = est.predict_instances(imgs, Ks, max_instances=M)
    est.stages.clear()
    _same(gp, wp, 'poses')
    _same_inter(got, want, f'M={M}')
    np.testing.assert_array_equal(got['instance_count'], [min(len(b), M) for b in boxes])
    assert np.isneginf(got['det_score'][1]).all() and not got['instance_valid'][1].any()


@pytest.mark.parametrize('kind', ['cuda', 'nv12', 'resized', 'two_sizes', 'cuda_boxes'])
def test_frame_kinds_and_cuda_boxes_equal_the_numpy_path(est, found, kind):
    imgs, Ks, boxes, _ = found
    ins, ref, bx = imgs, imgs, boxes
    if kind == 'two_sizes':
        ref = _two_sizes(imgs, range(3))
        ins = [torch.from_numpy(im).cuda() for im in ref]
    elif kind == 'cuda_boxes':
        bx = [torch.from_numpy(b).cuda() for b in boxes]
    else:
        ins, ref = _inputs(kind, imgs)
    gp, got = est.predict_instances(ins, Ks, max_instances=2, boxes=bx)
    wp, want = est.predict_instances(ref, Ks, max_instances=2, boxes=boxes)
    _same(gp, wp, kind)
    _same_inter(got, want, kind)


def test_predict_batch_is_one_instance(est, found):
    imgs, Ks, boxes, _ = found
    one = [b[0] for b in boxes]
    p, inter = est.predict_batch(imgs, Ks, boxes=one)
    wp, want = est.predict_instances(imgs, Ks, max_instances=1, boxes=[b[None] for b in one])
    _same(p, wp[:, 0], 'poses')
    for k in ('det_position', 'det_scale_r2q', 'det_score', 'det_que_img', 'sel_angle_r2q', 'sel_scores', 'sel_ref_idx'):
        _same(inter[k], want[k][:, 0], k)
    for a, b in zip(inter['refine_poses'], want['refine_poses']):
        _same(a, b[:, 0], 'refine_poses')
    pc, ic = est.predict_batch(imgs, Ks, boxes=torch.from_numpy(np.stack(one)).cuda())     # CUDA boxes, one per frame
    _same(pc, p, 'cuda boxes')
    bad = np.stack(one)
    bad[1, 2] = bad[1, 0]                                                                  # degenerate
    pb, ib = est.predict_batch(imgs, Ks, boxes=torch.from_numpy(bad).cuda())
    assert np.isneginf(ib['det_score'][1]) and ib['det_scale_r2q'][1] == 1
    with pytest.raises(ValueError):
        est.predict_batch(imgs, Ks, boxes=bad)
    with pytest.raises(ValueError, match='exactly one box'):
        est.predict_batch(imgs, Ks, boxes=[b[:2] for b in boxes])


def test_round_trip_through_the_detector_records(est, found):
    """Boxes made from predict_instances' own records (squares of side 128 * scale) give the same instances, positions and
    scales to float32 rounding, the same selected views, and refinement chains near the detector path's.  The box
    corners round the records by about an ulp, which moves the crops by ~1e-5 px and flips single crop pixels; the
    refiner amplifies that, so the chains are held to a bar of that size rather than to the fp-order bar."""
    imgs, Ks, boxes, inter = found
    _, got = est.predict_instances(imgs, Ks, max_instances=2, boxes=boxes)
    valid = inter['instance_valid']
    _same(got['instance_valid'], valid, 'valid')
    _same(got['sel_ref_idx'][valid], inter['sel_ref_idx'][valid], 'selected view')
    np.testing.assert_allclose(got['det_position'][valid], inter['det_position'][valid], atol=1e-3)
    np.testing.assert_allclose(got['det_scale_r2q'][valid], inter['det_scale_r2q'][valid], rtol=1e-5)
    a, b = (np.stack([np.asarray(c[valid], np.float64) for c in r['refine_poses']]) for r in (got, inter))
    dev = np.abs(a - b).reshape(len(a), -1).max(1)
    print('round trip max |dpose| per iteration', dev)
    assert dev[0] < 2e-3 and (dev[1:] < 0.15).all(), dev


def test_object_set(est, db, found, monkeypatch):
    from gen6d_b200.synthetic import synthetic_database
    imgs, Ks, boxes, _ = found
    one = est.object_set()
    one.add('a', db)
    gp, got = one.predict_instances(imgs, Ks, max_instances=2, boxes=[{'a': b} for b in boxes])['a']
    wp, want = est.predict_instances(imgs, Ks, max_instances=2, boxes=boxes)
    _same(gp, wp, 'K = 1')
    _same_inter(got, want, 'K = 1')
    two = est.object_set()
    two.add('a', db)
    two.add('b', synthetic_database(seed=8))
    res = two.predict_instances(imgs, Ks, max_instances=2, boxes=[{'b': b} for b in boxes])
    np.testing.assert_array_equal(res['a'][1]['instance_count'], 0)
    np.testing.assert_array_equal(res['b'][1]['instance_count'], [len(b) for b in boxes])
    with pytest.raises(ValueError, match='not in the set'):
        two.predict_instances(imgs, Ks, boxes=[{'c': b} for b in boxes])


# ------------------------------------------------------------------------------------------ instance trackers
def test_lockstep_box_steps_equal_the_twin_detection(est, videos, found, monkeypatch):
    _, _, boxes, _ = found
    S, M = 3, 2
    a = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=None)
    imgs, Ks = _frames(videos, 0, S)
    first = a.step(imgs, Ks, boxes=boxes)
    _, want = est.predict_instances(imgs, Ks, max_instances=M, boxes=boxes)
    for k in KEYS:
        _same(first[3][k], want[k], k)
    rest = [a.step(*_frames(videos, t, S)) for t in range(1, 4)]
    est.stages.clear()
    _twin_detection(monkeypatch, est, _host_table(B.for_frames(boxes, S, 'x', 'cuda:0')), M)
    b = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=None)
    for t, g in enumerate([first] + rest):
        w = b.step(*_frames(videos, t, S))
        for x, y, k in zip(g[:3], w[:3], ('poses', 'smoothed', 'ids')):
            _same(x, y, f'step {t} {k}')
        _same_inter(g[3], w[3], f'step {t}')
    est.stages.clear()


def _centre_boxes(trk, poses, ids, Ks, side):
    """A box of side `side` at every live track's projected object centre, per sequence."""
    c = np.asarray(trk.est.ref_info['center'], np.float64).reshape(3)
    out = []
    for s in range(len(poses)):
        rows = []
        for m in range(poses.shape[1]):
            if ids[s, m] < 0:
                continue
            p = Ks[s] @ (poses[s, m, :, :3].astype(np.float64) @ c + poses[s, m, :, 3])
            x, y = p[:2] / p[2]
            rows.append([x - side / 2, y - side / 2, x + side / 2, y + side / 2, 1.0])
        out.append(np.asarray(rows, np.float32).reshape(-1, 5))
    return out


def test_boxes_keep_ids_and_empty_boxes_drop_tracks(est, videos, found):
    _, _, boxes, _ = found
    S, M = 3, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, max_misses=1)
    p, _, ids, _ = trk.step(*_frames(videos, 0, S), boxes=boxes)
    assert (ids >= 0).sum() == sum(len(b) for b in boxes)
    imgs, Ks = _frames(videos, 1, S)
    side = 128.0 * float(np.median(found[3]['det_scale_r2q'][found[3]['instance_valid']]))
    p2, _, ids2, inter = trk.step(imgs, Ks, boxes=_centre_boxes(trk, p, ids, np.stack(Ks), side))
    _same(ids2, ids, 'ids kept')
    assert not inter['spawned'].any() and inter['dropped'] == []
    empty = [np.zeros((0, 4), np.float32)] * S
    _, _, ids3, inter3 = trk.step(*_frames(videos, 2, S), boxes=empty)
    _same(ids3, ids, 'one miss keeps the tracks')
    assert (trk._state['misses'].cpu().numpy()[trk._state['live'].cpu().numpy() != 0] == 1).all()
    _, _, ids4, inter4 = trk.step(*_frames(videos, 3, S), boxes=empty)
    assert (ids4 < 0).all() and inter4['dropped'] == sorted(int(i) for i in ids[ids >= 0])


def test_per_sequence_box_steps(est, videos, found):
    _, _, boxes, _ = found
    S, M = 3, 2
    trk = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=2, schedule='per_sequence')
    ref = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=None)
    imgs, Ks = _frames(videos, 0, S)
    _same_inter(trk.step(imgs, Ks, boxes=boxes)[3], ref.step(imgs, Ks, boxes=boxes)[3] | {'detected': np.ones(S, bool)},
                'first step')
    imgs, Ks = _frames(videos, 1, S)
    trk.step(imgs, Ks), ref.step(imgs, Ks)
    assert trk.detecting().all()                                                   # every sequence due (E = 2)
    imgs, Ks = _frames(videos, 2, S)
    p, sm, ids, inter = trk.step(imgs, Ks, boxes=[boxes[0], None, None])
    assert inter['detected'].tolist() == [True, False, False]
    assert trk.detecting().tolist() == [False, True, True]                        # unboxed due sequences stay due
    _, want = est.predict_instances([imgs[0]], [Ks[0]], max_instances=M, boxes=[boxes[0]])
    for k in KEYS:
        _same(inter[k][:1], want[k], k)
    rp, rsm, rids, _ = ref.step(imgs, Ks)                                          # the others: a refine step
    for s in (1, 2):
        _same(ids[s], rids[s], f'ids {s}')
        _same(p[s], rp[s], f'poses {s}')
        _same(sm[s], rsm[s], f'smoothed {s}')
    # a partial step, boxes in sequences= order
    p, _, _, inter = trk.step([imgs[2], imgs[1]], [Ks[2], Ks[1]], sequences=[2, 1], boxes=[None, boxes[1]])
    assert inter['detected'].tolist() == [False, True] and trk.detecting().tolist() == [False, False, True]


def test_drawing_and_out_on_box_steps(est, videos, found):
    _, _, boxes, _ = found
    S = 3
    a = est.instance_tracker(num_sequences=S, max_instances=2, draw='raw')
    b = est.instance_tracker(num_sequences=S, max_instances=2)
    imgs, Ks = _frames(videos, 0, S)
    out = {'raw': [torch.zeros_like(torch.from_numpy(im)).cuda() for im in imgs]}
    ga, gb = a.step(imgs, Ks, out=out, boxes=boxes), b.step(imgs, Ks, boxes=boxes)
    for x, y, k in zip(ga[:3], gb[:3], ('poses', 'smoothed', 'ids')):
        _same(x, y, k)
    for s in range(S):
        drawn = out['raw'][s].cpu().numpy()
        assert (drawn != imgs[s]).any() and (drawn == imgs[s]).mean() > 0.5
    ga2 = a.step(imgs, Ks, boxes=boxes)
    assert len(ga2[3]['drawn']['raw']) == S


def test_object_instance_tracker_k1_equals_estimator(est, db, videos, found):
    _, _, boxes, _ = found
    S = 3
    objs = est.object_set()
    objs.add('a', db)
    a = objs.instance_tracker(num_sequences=S, max_instances=2, schedule='per_sequence', redetect_every=3)
    b = est.instance_tracker(num_sequences=S, max_instances=2, schedule='per_sequence', redetect_every=3)
    for t in range(4):
        imgs, Ks = _frames(videos, t, S)
        bx = [boxes[s] if (t + s) % 2 == 0 else None for s in range(S)]
        g, w = a.step(imgs, Ks, boxes=[None if x is None else {'a': x} for x in bx])['a'], b.step(imgs, Ks, boxes=bx)
        for x, y, k in zip(g[:3], w[:3], ('poses', 'smoothed', 'ids')):
            _same(x, y, f'step {t} {k}')
        _same_inter(g[3], w[3], f'step {t}')
