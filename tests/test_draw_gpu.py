"""Drawn frames (row f16) on the H100: g6d_draw_boxes against its host twin on every byte, and a drawing tracker's frames
against predict.py's draw_bbox_3d on live cv2 with the step's own poses, its results against a non-drawing tracker's."""
import os

import cv2
import numpy as np
import pytest
import torch

from test_draw_cpu import cv_draw_bbox_3d, host_draw, nv12_of, project, random_case

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))


def _pitched(img, pad=7):
    h, w = img.shape[:2]
    big = torch.randint(0, 256, (h + 3, w + 2 + pad, 3), dtype=torch.uint8, device='cuda')
    big[1:1 + h, 2:2 + w] = torch.from_numpy(img).cuda()
    return big[1:1 + h, 2:2 + w]


def _nv12_dst(h, w, pad=5):
    from gen6d_b200.frames import NV12
    surf = torch.randint(0, 256, (h * 3 // 2, w + pad), dtype=torch.uint8, device='cuda')
    return NV12(surf[:h, :w], surf[h:, :w])


def test_kernel_equals_host_twin():
    """Frames of mixed sizes (pitched sources), up to 16 boxes each at both precisions, into contiguous RGB, pitched RGB
    and NV12 destinations."""
    from gen6d_b200 import draw as dr
    rng = np.random.RandomState(1)
    sizes = [(48, 64), (31, 17), (2, 2), (1, 40), (60, 60), (40, 1)]
    imgs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    Ks, poses, wants, outs = [], [], [], []
    bbox = (rng.randn(8, 3) * 0.5).astype(np.float32)
    for i, (img, (h, w)) in enumerate(zip(imgs, sizes)):
        n = [1, 3, 16, 2, 7, 1][i]
        f32 = i % 2 == 0
        ps, K = [], None
        for _ in range(n):
            p, K0, _ = random_case(rng, h, w, f32)
            K = K0 if K is None else K
            ps.append(p)
        Ks.append(K)
        poses.append(np.stack(ps).astype(np.float32 if f32 else np.float64))
        wants.append(host_draw(img, [(p, f32, K, bbox, (0, 0, 255)) for p in ps]))
    frames = [_pitched(im, 3 + i) for i, im in enumerate(imgs)]
    got = dr.draw_boxes(frames, Ks, poses, bbox)
    for i, (g, w_) in enumerate(zip(got, wants)):
        np.testing.assert_array_equal(g.cpu().numpy(), w_, err_msg=f'frame {i}')
    out = [_pitched(np.zeros_like(im), 9) if (h % 2 or w % 2) else _nv12_dst(h, w) for im, (h, w) in zip(imgs, sizes)]
    dr.draw_boxes(frames, Ks, poses, bbox, out=out)
    for i, (o, w_) in enumerate(zip(out, wants)):
        if isinstance(o, torch.Tensor):
            np.testing.assert_array_equal(o.cpu().numpy(), w_, err_msg=f'frame {i}')
        else:
            wy, wuv = nv12_of(w_)
            np.testing.assert_array_equal(o.y.cpu().numpy(), wy, err_msg=f'frame {i} Y')
            np.testing.assert_array_equal(o.uv.cpu().numpy(), wuv, err_msg=f'frame {i} UV')


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    e, db = build_estimator()
    e.cfg['device_glue'] = True
    return e, db


@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K'].astype(np.float32)
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _strip(inter):
    return {k: v for k, v in inter.items() if k != 'drawn'}


def _same(got, want, where=''):
    if isinstance(want, dict):
        assert set(got) == set(want), where
        for k in want:
            _same(got[k], want[k], f'{where}.{k}')
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f'{where}[{i}]')
    else:
        g, w = np.asarray(got), np.asarray(want)
        assert g.dtype == w.dtype and g.shape == w.shape, where
        np.testing.assert_array_equal(g, w, err_msg=where)


def _kernels(tracker):
    return sorted(st.kernels for st in tracker.stages.stages.values())


@pytest.mark.parametrize('inputs', ['numpy', 'cuda', 'nv12'])
def test_tracker_draws_predict_py_frames(est, video, inputs):
    """Full, refine, mixed (reset) and refine steps: every drawn frame is draw_bbox_3d on live cv2 with the step's own
    raw (float32) and smoothed (float64) poses, the results equal a non-drawing tracker's, each drawing graph holds the
    non-drawing graph's kernels plus the draw node, and new destinations replay the same graphs."""
    from gen6d_b200.frames import NV12
    e, _ = est
    frames, K = video
    S = 2
    dt, nt = e.tracker(num_sequences=S, draw=('raw', 'smoothed')), e.tracker(num_sequences=S)
    bbox = dt.bbox
    for t in range(5):
        if t == 3:
            dt.reset([1])
            nt.reset([1])
        imgs = [np.ascontiguousarray(frames[(t + s) % len(frames)]) for s in range(S)]
        if inputs == 'numpy':
            ins = imgs
        elif inputs == 'cuda':
            ins = [_pitched(im, 5 + s) for s, im in enumerate(imgs)]
        else:
            ins = []
            for im in imgs:
                y, uv = nv12_of(im)
                ins.append(NV12(torch.from_numpy(y).cuda(), torch.from_numpy(uv).cuda()))
                im[...] = cv2.cvtColor(np.vstack([y, uv]), cv2.COLOR_YUV2RGB_NV12)      # the working frame the graph holds
        Ks = [K] * S
        raw, smoothed, inter = dt.step(ins, Ks)
        want = nt.step(imgs if inputs == 'numpy' else ins, Ks)
        _same((raw, smoothed, _strip(inter)), want, f'step {t}')
        for s in range(S):
            r = cv_draw_bbox_3d(imgs[s], project(bbox, raw[s], K), (0, 0, 255))
            m = cv_draw_bbox_3d(imgs[s], project(bbox, smoothed[s], K), (0, 0, 255))
            np.testing.assert_array_equal(inter['drawn']['raw'][s].cpu().numpy(), r, err_msg=f'step {t} raw {s}')
            np.testing.assert_array_equal(inter['drawn']['smoothed'][s].cpu().numpy(), m, err_msg=f'step {t} smoothed {s}')
    assert [k + 1 for k in _kernels(nt)] == _kernels(dt)
    # out=: caller destinations (pitched RGB and NV12), written inside the graph; new allocations replay the same graph
    n = len(dt.stages.stages)
    for t in range(2):
        h, w = frames[0].shape[:2]
        out = {'raw': [_pitched(np.zeros((h, w, 3), np.uint8), 3 + t) for _ in range(S)],
               'smoothed': [_nv12_dst(h, w, 2 + t) for _ in range(S)]}
        imgs = [np.ascontiguousarray(frames[(t + s) % len(frames)]) for s in range(S)]
        ins = imgs if inputs == 'numpy' else [_pitched(im, 1) for im in imgs]
        raw, smoothed, inter = dt.step(ins, [K] * S, out=out)
        assert 'drawn' not in inter
        for s in range(S):
            np.testing.assert_array_equal(out['raw'][s].cpu().numpy(), cv_draw_bbox_3d(imgs[s], project(bbox, raw[s], K), (0, 0, 255)))
            wy, wuv = nv12_of(cv_draw_bbox_3d(imgs[s], project(bbox, smoothed[s], K), (0, 0, 255)))
            np.testing.assert_array_equal(out['smoothed'][s].y.cpu().numpy(), wy)
            np.testing.assert_array_equal(out['smoothed'][s].uv.cpu().numpy(), wuv)
    assert len(dt.stages.stages) == n


def test_tracker_draw_errors(est, video):
    e, _ = est
    frames, K = video
    t = e.tracker(num_sequences=1, draw='smoothed')
    h, w = frames[0].shape[:2]
    with pytest.raises(ValueError, match='exactly the drawn kinds'):
        t.step([frames[0]], [K], out={'raw': [torch.zeros(h, w, 3, dtype=torch.uint8, device='cuda')]})
    with pytest.raises(ValueError, match='one per sequence'):
        t.step([frames[0]], [K], out={'smoothed': []})
    with pytest.raises(ValueError, match='working size'):
        t.step([frames[0]], [K], out={'smoothed': [torch.zeros(h + 1, w, 3, dtype=torch.uint8, device='cuda')]})
    with pytest.raises(ValueError, match='create the tracker with draw='):
        e.tracker(num_sequences=1).step([frames[0]], [K], out={'smoothed': [None]})
    with pytest.raises(ValueError, match='draw must be'):
        e.tracker(num_sequences=1, draw='both')
    was = e.cfg['device_glue']
    e.cfg['device_glue'] = False
    try:
        with pytest.raises(ValueError, match='device pipeline'):
            e.tracker(num_sequences=1, draw='raw').step([frames[0]], [K])
    finally:
        e.cfg['device_glue'] = was


# ------------------------------------------------------------------------------------------ the other trackers
@pytest.fixture(scope='module')
def objs(est):
    from gen6d_b200.synthetic import synthetic_database
    e, db = est
    o = e.object_set()
    o.add('a', db)
    o.add('b', synthetic_database(seed=8))
    return o


def _mixed_sizes(frames, t, S):
    """S numpy frames of the video, every second one cropped: a step over frames of different sizes (the canvas)."""
    out = []
    for s in range(S):
        f = np.ascontiguousarray(frames[(t + s) % len(frames)])
        out.append(np.ascontiguousarray(f[:400, :600]) if s % 2 else f)
    return out


def _drawn(img, boxes):
    """draw_bbox_3d applied box after box: boxes [(bbox, pose, K, colour)]."""
    for bbox, pose, K, color in boxes:
        img = cv_draw_bbox_3d(img, project(bbox, pose, K), color)
    return img


def _check_frames(drawn, imgs, want_boxes, where):
    for kind, per_seq in want_boxes.items():
        for s, boxes in enumerate(per_seq):
            np.testing.assert_array_equal(drawn[kind][s].cpu().numpy(), _drawn(imgs[s], boxes), err_msg=f'{where} {kind} {s}')


def test_tracker_single_kind_resized(est, video):
    """draw='smoothed' only (destination s, smoothed pose row s) on Resized NV12 frames: the drawn frame is draw_bbox_3d on
    cv2's working frame, the results equal a numpy tracker's on those frames."""
    from gen6d_b200.frames import NV12, Resized
    e, _ = est
    frames, K = video
    S = 2
    dt, nt = e.tracker(num_sequences=S, draw='smoothed'), e.tracker(num_sequences=S)
    pt = e.tracker(num_sequences=S)                  # the same Resized feed without drawing: its graphs' kernel counts
    for t in range(4):
        if t == 2:
            for tr in (dt, nt, pt):
                tr.reset([0])
        ins, work = [], []
        for s in range(S):
            img = np.ascontiguousarray(frames[(t + s) % len(frames)])
            big = cv2.resize(img, (1280, 960), interpolation=cv2.INTER_CUBIC)
            y, uv = nv12_of(big)
            ins.append(Resized(NV12(torch.from_numpy(y).cuda(), torch.from_numpy(uv).cuda()), max_side=640))
            rgb = cv2.cvtColor(np.vstack([y, uv]), cv2.COLOR_YUV2RGB_NV12)
            work.append(cv2.resize(rgb, (640, 480), interpolation=cv2.INTER_LINEAR))
        raw, smoothed, inter = dt.step(ins, [K] * S)
        _same((raw, smoothed, _strip(inter)), nt.step(work, [K] * S), f'step {t}')
        pt.step(ins, [K] * S)
        assert set(inter['drawn']) == {'smoothed'}
        _check_frames(inter['drawn'], work, {'smoothed': [[(dt.bbox, smoothed[s], K, (0, 0, 255))] for s in range(S)]}, f'step {t}')
    assert [k + 1 for k in _kernels(pt)] == _kernels(dt)


def test_object_tracker_draws_every_object(objs, video):
    """Every object's box on its sequence's frame in object order (own colours), frames of different sizes (the canvas
    sources), full, refine, mixed and refine steps."""
    frames, K = video
    S, colors = 3, {'a': (0, 0, 255), 'b': (0, 255, 0)}
    dt, nt = objs.tracker(num_sequences=S, draw=('raw', 'smoothed'), draw_colors={'b': (0, 255, 0)}), objs.tracker(num_sequences=S)
    for t in range(4):
        if t == 2:
            dt.reset([1])
            nt.reset([1])
        imgs = _mixed_sizes(frames, t, S)
        got, want = dt.step(imgs, [K] * S), nt.step(imgs, [K] * S)
        _same({n: (r, m, _strip(i)) for n, (r, m, i) in got.items()}, want, f'step {t}')
        drawn = got['a'][2]['drawn']
        assert all(v[2]['drawn'] is drawn for v in got.values())
        boxes = {'raw': [[(dt.bboxes[o], got[n][0][s], K, colors[n]) for o, n in enumerate(objs.names)] for s in range(S)],
                 'smoothed': [[(dt.bboxes[o], got[n][1][s], K, colors[n]) for o, n in enumerate(objs.names)] for s in range(S)]}
        _check_frames(drawn, imgs, boxes, f'step {t}')
    assert [k + 1 for k in _kernels(nt)] == _kernels(dt)


def _instance_boxes(res, bboxes, names, colors, K, S, M, kind):
    """Per sequence the live slots' boxes in row order (slot m, then object)."""
    k = 0 if kind == 'raw' else 1
    return [[(bboxes[o], res[n][k][s, m], K, colors[n]) for m in range(M) for o, n in enumerate(names) if res[n][2][s, m] >= 0]
            for s in range(S)]


def test_instance_trackers_draw_live_slots(est, objs, video):
    """est.instance_tracker and objs.instance_tracker: only live slots (track id >= 0) are drawn, in slot order; detect and
    refine steps, results equal a non-drawing tracker's, one more C-ABI kernel per graph, out= replays the same graph."""
    from gen6d_b200.frames import NV12
    e, _ = est
    frames, K = video
    S, M = 2, 2
    cases = [(lambda **k: e.instance_tracker(num_sequences=S, max_instances=M, **k), ['obj'], {'obj': (0, 0, 255)}, {}),
             (lambda **k: objs.instance_tracker(num_sequences=S, max_instances=M, **k), objs.names,
              {'a': (0, 0, 255), 'b': (255, 255, 0)}, {'draw_colors': {'b': (255, 255, 0)}})]
    for make, names, colors, kw in cases:
        dt, nt = make(draw=('raw', 'smoothed'), **kw), make()
        bboxes = [dt.bboxes[o] for o in range(len(names))] if hasattr(dt, 'names') else [dt.bbox]
        n_live = 0
        for t in range(5):
            if t == 3:
                dt.redetect()
                nt.redetect()
            imgs = _mixed_sizes(frames, t, S) if t < 4 else [np.ascontiguousarray(frames[(t + s) % len(frames)]) for s in range(S)]
            got, want = dt.step(imgs, [K] * S), nt.step(imgs, [K] * S)
            if not hasattr(dt, 'names'):
                got, want = {'obj': got}, {'obj': want}
            _same({n: (*v[:3], _strip(v[3])) for n, v in got.items()}, want, f'step {t}')
            drawn = got[names[0]][3]['drawn']
            n_live += sum(int((got[n][2] >= 0).sum()) for n in names)
            _check_frames(drawn, imgs, {kd: _instance_boxes(got, bboxes, names, colors, K, S, M, kd) for kd in ('raw', 'smoothed')},
                          f'step {t}')
        assert n_live > 0
        assert [k + 1 for k in _kernels(nt)] == _kernels(dt)
        n = len(dt.stages.stages)
        h, w = frames[0].shape[:2]
        out = {'raw': [_pitched(np.zeros((h, w, 3), np.uint8), 4) for _ in range(S)], 'smoothed': [_nv12_dst(h, w, 3) for _ in range(S)]}
        imgs = [np.ascontiguousarray(frames[s]) for s in range(S)]
        got = dt.step(imgs, [K] * S, out=out)
        if not hasattr(dt, 'names'):
            got = {'obj': got}
        for s in range(S):
            np.testing.assert_array_equal(out['raw'][s].cpu().numpy(),
                                          _drawn(imgs[s], _instance_boxes(got, bboxes, names, colors, K, S, M, 'raw')[s]))
            wy, wuv = nv12_of(_drawn(imgs[s], _instance_boxes(got, bboxes, names, colors, K, S, M, 'smoothed')[s]))
            np.testing.assert_array_equal(out['smoothed'][s].y.cpu().numpy(), wy)
            np.testing.assert_array_equal(out['smoothed'][s].uv.cpu().numpy(), wuv)
        assert len(dt.stages.stages) == n
