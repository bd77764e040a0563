"""Several objects per frame (gen6d_b200/objects.py) on the H100: the object-major correlation regroup kernel, one object
against predict_batch bit for bit, three objects against three single-object estimators, one query pyramid and one graph
per call, isolation from the estimator's own object, membership changes, staleness and the errors."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENS = np.load(os.path.join(HERE, 'golden', 'sens_golden.npz'))
SEEDS = {'a': 7, 'b': 8, 'c': 11}
KEYS = ('det_position', 'det_scale_r2q', 'det_que_img', 'sel_ref_idx', 'sel_angle_r2q', 'sel_scores')


@pytest.fixture(scope='module')
def dbs():
    from gen6d_b200.synthetic import synthetic_database
    return {n: synthetic_database(seed=s) for n, s in SEEDS.items()}


@pytest.fixture(scope='module')
def frames6(dbs):
    """2 frames from each database."""
    imgs, Ks = [], []
    for db in dbs.values():
        for i in db.get_img_ids()[:2]:
            imgs.append(db.get_image(i))
            Ks.append(db.get_K(i))
    return imgs, Ks


@pytest.fixture(scope='module')
def est(dbs):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(dbs['a'])[0]


def _single(db):
    from gen6d_b200.synthetic import build_estimator
    return build_estimator(db)[0]


def _single_results(e, imgs, Ks):
    """predict_batch of a single-object estimator, its captured graph's kernel count and its raw correlation maps."""
    from gen6d_b200 import ops
    poses, inter = e.predict_batch(imgs, Ks)
    kernels = sum(s.kernels for s in e.stages.stages.values())
    with torch.no_grad():
        u8 = e.detector.upload_frame([np.asarray(f) for f in imgs])
        raw = e.detector._detect_nhwc(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False), return_taps=True)['raw']
        raw = [[m.cpu().numpy() for m in scale] for scale in raw]
    return {'poses': poses, 'inter': inter, 'kernels': kernels, 'raw': raw}


@pytest.fixture(scope='module')
def singles(dbs, frames6):
    """Per object, a single-object estimator built on its database, on the same 6 frames (plus 5 frames of 'a')."""
    out = {}
    e = None
    for n, db in dbs.items():
        if e is None:
            e = _single(db)
        else:
            e.build(db, 'all')
        out[n] = _single_results(e, *frames6)
        if n == 'a':
            ids = db.get_img_ids()[:5]
            out['a5'] = e.predict_batch([db.get_image(i) for i in ids], [db.get_K(i) for i in ids])
    return out


@pytest.fixture(scope='module')
def objs3(est, dbs):
    objs = est.object_set()
    for n, db in dbs.items():
        objs.add(n, db)
    return objs


def _assert_matches_single(got, want, name):
    """The bars of three objects against a single-object estimator on the same frames."""
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
    print(name, 'object set vs single-object predict_batch, max |dpose| per iteration', dev)
    assert dev[0] < 1e-4, (name, dev)
    assert (dev[1:] <= np.maximum(2.0 * SENS['gain_R'][1:] * 1e-3, 2e-3)).all(), (name, dev)
    np.testing.assert_array_equal(poses, inter['refine_poses'][-1])


def _assert_same(a, b):
    for name in a:
        (pa, ia), (pb, ib) = a[name], b[name]
        np.testing.assert_array_equal(pa, pb, err_msg=name)
        for k in KEYS + ('det_score',):
            np.testing.assert_array_equal(ia[k], ib[k], err_msg=f'{name} {k}')
        for x, y in zip(ia['refine_poses'], ib['refine_poses']):
            np.testing.assert_array_equal(x, y, err_msg=name)


# ------------------------------------------------------------------------------------------ 1. the kernel
@pytest.mark.parametrize('rfn', [4, 32])
@pytest.mark.parametrize('qn', [1, 2])
@pytest.mark.parametrize('n_obj', [1, 3])
@pytest.mark.parametrize('k', [1, 3, 15])
def test_corr_rowsum_objects_kernel(k, n_obj, qn, rfn):
    from gen6d_b200 import ops
    H, W = 9, 7
    g = torch.Generator().manual_seed(1000 * k + 100 * n_obj + 10 * qn + rfn)
    partial = torch.randn(qn, H + k - 1, W, n_obj * k * rfn, generator=g).cuda()
    got = ops.det_corr_rowsum_objects(partial, n_obj, k, rfn)
    assert got.shape == (n_obj, qn, H, W, rfn)
    want = torch.empty_like(got)
    for o in range(n_obj):
        acc = torch.zeros(qn, H, W, rfn, device='cuda')
        for ky in range(k):
            acc = acc + partial[:, ky:ky + H, :, (o * k + ky) * rfn:(o * k + ky + 1) * rfn]
        want[o] = acc
    np.testing.assert_array_equal(got.cpu().numpy(), want.cpu().numpy())
    if n_obj == 1:
        np.testing.assert_array_equal(got[0].cpu().numpy(), ops.det_corr_rowsum(partial, k, rfn).cpu().numpy())


# ------------------------------------------------------------------------------------------ 2. one object
def test_one_object_equals_predict_batch(est, dbs, singles):
    db = dbs['a']
    ids = db.get_img_ids()[:5]
    objs = est.object_set()
    objs.add('a', db)
    res = objs.predict([db.get_image(i) for i in ids], [db.get_K(i) for i in ids])
    assert list(res) == ['a']
    poses, inter = res['a']
    wposes, want = singles['a5']
    np.testing.assert_array_equal(poses, wposes)
    for k in KEYS:
        np.testing.assert_array_equal(inter[k], want[k], err_msg=k)
        assert inter[k].dtype == want[k].dtype and inter[k].shape == want[k].shape, k
    assert len(inter['refine_poses']) == len(want['refine_poses'])
    for x, y in zip(inter['refine_poses'], want['refine_poses']):
        assert x.dtype == y.dtype
        np.testing.assert_array_equal(x, y)
    assert inter['det_score'].shape == (5,) and np.isfinite(inter['det_score']).all()


# ------------------------------------------------------------------------------------------ 3. three objects
def test_three_objects_equal_three_estimators(objs3, frames6, singles):
    res = objs3.predict(*frames6)
    assert list(res) == ['a', 'b', 'c']
    for n in res:
        _assert_matches_single(res[n], (singles[n]['poses'], singles[n]['inter']), n)
        assert res[n][1]['det_score'].shape == (6,)
    raw = objs3.raw_correlation(frames6[0])
    worst = 0.0
    for n in res:
        for got_s, want_s in zip(raw[n], singles[n]['raw']):
            for got, want in zip(got_s, want_s):
                got = got.cpu().numpy()
                assert got.shape == want.shape
                rel = float(np.abs(got - want).max() / np.abs(want).max())
                worst = max(worst, rel)
    print('raw correlation maps, object set vs single object, max relative difference', worst)
    assert worst <= 3e-5


# ------------------------------------------------------------------------------------------ 4. one pyramid
def test_query_pyramid_runs_once(objs3, est, frames6, monkeypatch):
    monkeypatch.setenv('G6D_GRAPHS', '0')
    det = est.detector
    calls = []
    orig = det._features

    def counting(x):
        calls.append(tuple(x.shape))
        return orig(x)
    monkeypatch.setattr(det, '_features', counting)
    objs3.predict(*frames6)
    assert len(calls) == len(det.cfg['detection_scales']) == 4, calls


# ------------------------------------------------------------------------------------------ 5. one graph
def test_one_graph_per_call(objs3, frames6, singles):
    from gen6d_b200.graphs import REPLAYED_KERNELS
    from gen6d_b200.network.base import IO_BYTES
    a = objs3.predict(*frames6)
    assert len(objs3.stages.stages) == 1
    stage = next(iter(objs3.stages.stages.values()))
    k0, d0 = REPLAYED_KERNELS[0], IO_BYTES['d2h']
    b = objs3.predict(*frames6)
    assert len(objs3.stages.stages) == 1 and next(iter(objs3.stages.stages.values())) is stage
    assert REPLAYED_KERNELS[0] - k0 == stage.kernels                  # one replay ...
    assert IO_BYTES['d2h'] - d0 == stage.static_out.numel()            # ... and one read
    _assert_same(a, b)
    total = sum(singles[n]['kernels'] for n in SEEDS)
    print('object set graph kernels', stage.kernels, 'vs three single-object graphs', total)
    assert stage.kernels < total


# ------------------------------------------------------------------------------------------ 6. isolation
def test_estimator_and_set_are_isolated(dbs, frames6):
    from gen6d_b200.synthetic import build_estimator, synthetic_database
    e, db = build_estimator(dbs['a'])
    ids = db.get_img_ids()[:4]
    imgs, Ks = [db.get_image(i) for i in ids], [db.get_K(i) for i in ids]
    before = e.predict_batch(imgs, Ks)
    objs = e.object_set()
    for n, d in dbs.items():
        objs.add(n, d)
    first = objs.predict(*frames6)
    after = e.predict_batch(imgs, Ks)
    np.testing.assert_array_equal(before[0], after[0])
    for k in KEYS:
        np.testing.assert_array_equal(before[1][k], after[1][k], err_msg=k)
    e.build(synthetic_database(seed=9), 'all')
    e.predict_batch(imgs, Ks)
    _assert_same(first, objs.predict(*frames6))


# ------------------------------------------------------------------------------------------ 7. membership and staleness
def test_membership_and_staleness(est, dbs, frames6, singles):
    from gen6d_b200.synthetic import synthetic_database
    objs = est.object_set()
    for n, d in dbs.items():
        objs.add(n, d)
    objs.remove('b')
    assert objs.names == ['a', 'c']
    res = objs.predict(*frames6)
    assert list(res) == ['a', 'c']
    for n in res:
        _assert_matches_single(res[n], (singles[n]['poses'], singles[n]['inter']), n)
    db12 = synthetic_database(seed=12)
    objs.add('b', db12)
    assert objs.names == ['a', 'c', 'b']
    res = objs.predict(*frames6)
    want = _single_results(_single(db12), *frames6)
    _assert_matches_single(res['b'], (want['poses'], want['inter']), 'b (seed 12)')
    # new weights (the same values: every stored reference feature is stale all the same)
    est.selector.load_state_dict(est.selector.state_dict())
    with pytest.raises(RuntimeError, match='stale'):
        objs.predict(*frames6)
    for n, d in (('a', dbs['a']), ('c', dbs['c']), ('b', db12)):
        objs.remove(n)
        objs.add(n, d)
    fresh = est.object_set()
    for n, d in (('a', dbs['a']), ('c', dbs['c']), ('b', db12)):
        fresh.add(n, d)
    _assert_same(objs.predict(*frames6), fresh.predict(*frames6))


# ------------------------------------------------------------------------------------------ 8. errors
def test_errors(est, dbs, frames6):
    import types
    from gen6d_b200.estimator import Gen6DEstimator
    from gen6d_b200.synthetic import synthetic_database
    objs = est.object_set()
    with pytest.raises(ValueError, match='empty'):
        objs.predict(*frames6)
    objs.add('a', dbs['a'])
    with pytest.raises(ValueError, match='already'):
        objs.add('a', dbs['b'])
    with pytest.raises(ValueError, match='not in the set'):
        objs.remove('x')
    with pytest.raises(ValueError, match='detector reference views'):
        objs.add('few', synthetic_database(n_views=20))
    assert objs.names == ['a']
    no_refiner = Gen6DEstimator({}, modules={'detector': est.detector, 'selector': est.selector})
    with pytest.raises(ValueError, match='refiner'):
        no_refiner.object_set()
    comm = est.selector.comm
    try:
        est.selector.comm = types.SimpleNamespace(world=2, capturable=False)
        with pytest.raises(ValueError, match='sharded'):
            est.object_set()
    finally:
        est.selector.comm = comm
    est.cfg['host_warps'] = True
    try:
        with pytest.raises(ValueError, match='host_warps'):
            est.object_set()
    finally:
        est.cfg['host_warps'] = False
