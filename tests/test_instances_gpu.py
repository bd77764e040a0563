"""Several instances per frame (Gen6DEstimator.predict_instances, ObjectSet.predict_instances) on the H100: M = 1 against
predict_batch / ObjectSet.predict bit for bit, instance 0 of M = 3 against predict_batch, every valid row against the
stages run on its own, the masks against the peak kernel, a frame with two copies of the object, one graph and one read
per call, two objects, and the errors."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENS = np.load(os.path.join(HERE, 'golden', 'sens_golden.npz'))
KEYS = ('det_position', 'det_scale_r2q', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores')
M3 = dict(max_instances=3, nms_iou=0.3, peak_radius=1)


@pytest.fixture(scope='module')
def dbs():
    from gen6d_b200.synthetic import synthetic_database
    return {'a': synthetic_database(seed=7), 'b': synthetic_database(seed=8)}


@pytest.fixture(scope='module')
def est(dbs):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(dbs['a'])[0]


@pytest.fixture(scope='module')
def frames6(dbs):
    db = dbs['a']
    ids = db.get_img_ids()[:6]
    return [db.get_image(i) for i in ids], [db.get_K(i) for i in ids]


@pytest.fixture(scope='module')
def batch6(est, frames6):
    return est.predict_batch(*frames6)


@pytest.fixture(scope='module')
def inst3(est, frames6):
    return est.predict_instances(*frames6, **M3)


def _pose_bound(a, b, name):
    """The sensitivity bar test_objects_gpu.py holds an object set to against predict_batch."""
    a = np.stack([np.asarray(p, np.float64) for p in a])
    b = np.stack([np.asarray(p, np.float64) for p in b])
    dev = np.abs(a - b).reshape(len(a), -1).max(1)
    print(name, 'max |dpose| per iteration', dev)
    assert dev[0] < 1e-4, (name, dev)
    assert (dev[1:] <= np.maximum(2.0 * SENS['gain_R'][1:] * 1e-3, 2e-3)).all(), (name, dev)


# ------------------------------------------------------------------------------------------ 1. M = 1
def test_one_instance_equals_predict_batch(est, frames6, batch6):
    poses, inter = est.predict_instances(*frames6, max_instances=1)
    wposes, want = batch6
    assert poses.shape == (6, 1, 3, 4) and poses.dtype == wposes.dtype
    np.testing.assert_array_equal(poses[:, 0], wposes)
    for k in KEYS:
        assert inter[k].shape[:2] == (6, 1), k
        assert inter[k].dtype == want[k].dtype, k
        np.testing.assert_array_equal(inter[k][:, 0], want[k], err_msg=k)
    assert len(inter['refine_poses']) == len(want['refine_poses'])
    for x, y in zip(inter['refine_poses'], want['refine_poses']):
        assert x.dtype == y.dtype
        np.testing.assert_array_equal(x[:, 0], y)
    assert inter['instance_valid'].shape == (6, 1) and inter['instance_valid'].all()
    np.testing.assert_array_equal(inter['instance_count'], np.ones(6))


def test_one_instance_object_set_equals_predict(est, dbs, frames6):
    objs = est.object_set()
    for n, d in dbs.items():
        objs.add(n, d)
    want = objs.predict(*frames6)
    got = objs.predict_instances(*frames6, max_instances=1)
    assert list(got) == list(want)
    for n in want:
        (p, i), (wp, w) = got[n], want[n]
        np.testing.assert_array_equal(p[:, 0], wp, err_msg=n)
        for k in KEYS + ('det_score',):
            np.testing.assert_array_equal(i[k][:, 0], w[k], err_msg=f'{n} {k}')
        for x, y in zip(i['refine_poses'], w['refine_poses']):
            np.testing.assert_array_equal(x[:, 0], y, err_msg=n)


# ------------------------------------------------------------------------------------------ 2. instance 0 of M = 3
def test_instance0_matches_predict_batch(inst3, batch6):
    poses, inter = inst3
    _, want = batch6
    assert poses.shape == (6, 3, 3, 4)
    for k in ('det_position', 'det_scale_r2q', 'det_que_img'):
        np.testing.assert_array_equal(inter[k][:, 0], want[k], err_msg=k)
    np.testing.assert_array_equal(inter['sel_ref_idx'][:, 0], want['sel_ref_idx'])
    np.testing.assert_allclose(inter['sel_scores'][:, 0], want['sel_scores'], atol=3e-4)
    _pose_bound([p[:, 0] for p in inter['refine_poses']], want['refine_poses'], 'instance 0 vs predict_batch')


# ------------------------------------------------------------------------------------------ 3. every valid row
def test_valid_rows_equal_their_own_stages(est, frames6, inst3):
    from gen6d_b200 import ops
    poses, inter = inst3
    imgs, Ks = frames6
    valid = inter['instance_valid']
    assert valid[:, 0].all()
    print('instance counts', inter['instance_count'])
    res = est.cfg['ref_resolution']
    rows = [(f, m) for f in range(6) for m in range(3) if valid[f, m]]
    with torch.no_grad():
        frames = est.detector.upload_frame([np.asarray(f) for f in imgs])
        for f, m in rows:
            det = torch.tensor([[*inter['det_position'][f, m], inter['det_scale_r2q'][f, m], inter['det_score'][f, m]]],
                               dtype=torch.float32, device='cuda')
            crop = ops.warp_affine_u8(ops.glue_detection_jobs(det, frames[f:f + 1].contiguous(), res), 1, res, res)
            np.testing.assert_array_equal(crop[0].cpu().numpy(), inter['det_que_img'][f, m], err_msg=str((f, m)))
            sel = est.selector.select_que_imgs(inter['det_que_img'][f, m][None])
            assert sel['ref_idx'][0] == inter['sel_ref_idx'][f, m], (f, m)
        # the refinement chains of the valid rows, host-sequenced from the same initial poses
        fr = torch.stack([frames[f] for f, _ in rows]).contiguous()
        p0 = np.stack([inter['refine_poses'][0][f, m] for f, m in rows])
        _, chain = est._refine_batch_host(fr, [np.asarray(Ks[f]) for f, _ in rows], p0, est.cfg['refine_iter'])
    got = [np.stack([c[f, m] for f, m in rows]) for c in inter['refine_poses']]
    _pose_bound(got, chain, 'valid rows vs host refinement')


# ------------------------------------------------------------------------------------------ 4. masks
def test_masks_match_peak_kernel(est, frames6, inst3):
    from gen6d_b200 import ops
    _, inter = inst3
    with torch.no_grad():
        u8 = est.detector.upload_frame([np.asarray(f) for f in frames6[0]])
        o = est.detector._detect_nhwc(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False))
        det, idx, valid, count = ops.det_parse_peaks(o['score_predict'], o['scale_predict'], o['offset_predict'], 3, 1, 0.3,
                                                     float(est.cfg['ref_resolution']))
    np.testing.assert_array_equal(inter['instance_valid'], valid.cpu().numpy().T.astype(bool))
    np.testing.assert_array_equal(inter['instance_count'], count.cpu().numpy())
    np.testing.assert_array_equal(inter['det_position'], np.swapaxes(det.cpu().numpy()[..., :2], 0, 1))
    # invalid rows repeat instance 0's detection
    for f in range(6):
        for m in range(inter['instance_count'][f], 3):
            np.testing.assert_array_equal(inter['det_position'][f, m], inter['det_position'][f, 0])


# ------------------------------------------------------------------------------------------ 5. two copies of the object
def test_two_rendered_copies(est, dbs):
    db = dbs['a']
    i = db.get_img_ids()[3]
    pose, K = db.poses[i].copy(), db.get_K(i)
    far = pose.copy()
    far[0, 3] += 220.0 * pose[2, 3] / K[0, 0]                       # the same view shifted ~220 px to the right
    near = pose.copy()
    near[0, 3] -= 120.0 * pose[2, 3] / K[0, 0]
    a, b = db.render(near, K), db.render(far, K)
    img = np.where((b != db._bg).any(-1, keepdims=True), b, a)
    poses, inter = est.predict_instances([img, img], [K, K], max_instances=4, nms_iou=0.3)
    assert poses.shape == (2, 4, 3, 4) and np.isfinite(poses).all()
    for k in KEYS + ('det_score',):
        assert np.isfinite(inter[k].astype(np.float64)).all(), k
    np.testing.assert_array_equal(inter['instance_count'], inter['instance_valid'].sum(1))
    assert (inter['instance_count'] >= 1).all()
    np.testing.assert_array_equal(poses[0], poses[1])                # the same frame twice: the same rows
    print('two copies: instance counts', inter['instance_count'], 'positions', inter['det_position'][0])


# ------------------------------------------------------------------------------------------ 6. one graph, one read
def test_one_graph_per_call(est, frames6):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    a = est.predict_instances(*frames6, **M3)
    keys = [k for k in est.stages.stages if k[0][0] == 'instances']
    stage = est.stages.stages[next(k for k in keys if k[0][1:] == (3, 1, float(np.float32(0.3)), None))]
    n_graphs = len(est.stages.stages)
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    b = est.predict_instances(*frames6, **M3)
    assert len(est.stages.stages) == n_graphs
    assert REPLAYED_KERNELS[0] - k0 == stage.kernels                  # one replay ...
    assert IO_BYTES['d2h'] - d0 == stage.static_out.numel()            # ... and one read
    np.testing.assert_array_equal(a[0], b[0])
    for k in KEYS + ('instance_valid', 'instance_count'):
        np.testing.assert_array_equal(a[1][k], b[1][k], err_msg=k)
    est.predict_instances(*frames6, max_instances=2, nms_iou=0.3)
    assert len(est.stages.stages) == n_graphs + 1
    est.predict_instances(*frames6, max_instances=3, nms_iou=0.5)
    assert len(est.stages.stages) == n_graphs + 2
    est.predict_instances(*frames6, max_instances=3, nms_iou=0.5)
    assert len(est.stages.stages) == n_graphs + 2
    print('predict_instances graph kernels (M = 3)', stage.kernels)


# ------------------------------------------------------------------------------------------ 7. two objects
def test_two_objects(est, dbs, frames6):
    objs = est.object_set()
    for n, d in dbs.items():
        objs.add(n, d)
    want = objs.predict(*frames6)
    got = objs.predict_instances(*frames6, max_instances=2)
    assert list(got) == ['a', 'b']
    for n in got:
        p, i = got[n]
        w = want[n][1]
        assert p.shape == (6, 2, 3, 4) and i['instance_valid'].shape == (6, 2)
        for k in ('det_position', 'det_scale_r2q', 'det_score', 'det_que_img'):
            np.testing.assert_array_equal(i[k][:, 0], w[k], err_msg=f'{n} {k}')
        np.testing.assert_array_equal(i['sel_ref_idx'][:, 0], w['sel_ref_idx'], err_msg=n)
        np.testing.assert_allclose(i['sel_scores'][:, 0], w['sel_scores'], atol=3e-4, err_msg=n)
        _pose_bound([r[:, 0] for r in i['refine_poses']], w['refine_poses'], f'object {n} instance 0 vs ObjectSet.predict')
        np.testing.assert_array_equal(i['instance_count'], i['instance_valid'].sum(1))
    assert len(objs.stages.stages) == 2
    objs.predict_instances(*frames6, max_instances=2)
    assert len(objs.stages.stages) == 2


# ------------------------------------------------------------------------------------------ 8. errors and staleness
def test_errors_and_staleness(est, dbs, frames6):
    import types
    from gen6d_b200.estimator import Gen6DEstimator
    for kw in (dict(max_instances=0), dict(max_instances=17), dict(nms_iou=-0.1), dict(nms_iou=1.5), dict(peak_radius=4),
               dict(min_score=float('nan'))):
        with pytest.raises(ValueError):
            est.predict_instances(*frames6, **kw)
    no_refiner = Gen6DEstimator({}, modules={'detector': est.detector, 'selector': est.selector})
    with pytest.raises(ValueError, match='refiner'):
        no_refiner.predict_instances(*frames6)
    comm = est.selector.comm
    try:
        est.selector.comm = types.SimpleNamespace(world=2, capturable=False)
        with pytest.raises(ValueError, match='sharded'):
            est.predict_instances(*frames6)
    finally:
        est.selector.comm = comm
    est.cfg['host_warps'] = True
    try:
        with pytest.raises(ValueError, match='host_warps'):
            est.predict_instances(*frames6)
    finally:
        est.cfg['host_warps'] = False
    objs = est.object_set()
    with pytest.raises(ValueError, match='empty'):
        objs.predict_instances(*frames6)
    objs.add('a', dbs['a'])
    with pytest.raises(ValueError):
        objs.predict_instances(*frames6, max_instances=17)
    first = est.predict_instances(*frames6, max_instances=2)
    est.selector.load_state_dict(est.selector.state_dict())           # new weights (same values): graphs and the set go stale
    with pytest.raises(RuntimeError, match='stale'):
        objs.predict_instances(*frames6, max_instances=2)
    est.build(dbs['a'], 'all')
    again = est.predict_instances(*frames6, max_instances=2)           # recaptured on the rebuilt state
    np.testing.assert_array_equal(first[0], again[0])
