"""The upper face of the drop-in boundary (SURVEY.md 8b), checked against what the UNMODIFIED reference
expects of it, as recorded in tests/golden/dropin_golden.json by tests/golden/make_golden_dropin.py:

 * the reference's estimator.py binds this package's networks when `network` resolves to
   gen6d_b200.network (what a user does: put gen6d_b200/network on the path as `network`, or
   `sys.modules['network'] = gen6d_b200.network` before importing estimator / eval / predict): every name
   it imports from `network` exists, and every call it makes on the three networks (constructors
   included, estimator.py:117-125,166-171,179-213) binds to our methods;
 * every method the reference estimator calls exists on our classes with the reference's parameter names,
   order and defaults;
 * `VolumeRefiner.load_ref_imgs(database, ids)` accepts a reference `BaseDatabase` as estimator.py:171
   passes it (no wrapper in user code), takes the object's centre / diameter / up vector from the
   reference's `dataset.database` free functions, and the refinement host geometry runs on it.  The
   reference package is replaced by a stand-in module whose free functions return what the reference
   computed for this database.
Runs in a subprocess so that the module swaps cannot leak into the other tests."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import inspect, json, sys, types
    import numpy as np
    sys.path.insert(0, %(root)r)
    GOLD = json.load(open(%(root)r + '/tests/golden/dropin_golden.json'))

    import gen6d_b200.network as ours
    sys.modules['network'] = ours                 # the swap a user makes
    import network
    for name in GOLD['estimator_imports']:        # `from network import name2network` in estimator.py
        assert getattr(network, name) is getattr(ours, name), name
    assert set(ours.name2network) >= {'detector', 'selector', 'refiner'}

    def default_repr(p):
        return None if p.default is inspect.Parameter.empty else repr(p.default)

    for key, want in GOLD['signatures'].items():
        name, m = key.split('.')
        got = [[p.name, default_repr(p)] for p in inspect.signature(getattr(ours.name2network[name], m)).parameters.values()]
        assert got[:len(want)] == want, (key, got, want)                 # same names, order, defaults ...
        assert all(d is not None for _, d in got[len(want):]), (key, got)   # ... extras are optional
    print('signatures ok:', len(GOLD['signatures']))

    for name, m, npos, kws in GOLD['estimator_calls']:
        sig = inspect.signature(getattr(ours.name2network[name], m))
        sig.bind(None, *([None] * npos), **{k: None for k in kws})     # raises TypeError if the call does not bind
    print('estimator calls bind:', len(GOLD['estimator_calls']))

    # the reference's dataset.database free functions, as computed by the reference for this database
    ref = GOLD['database']
    def _lookup(key):
        def fn(database):
            assert database.database_name == ref['database_name'], database.database_name
            return np.asarray(ref[key], np.float32) if isinstance(ref[key], list) else ref[key]
        return fn
    dataset = types.ModuleType('dataset')
    dataset.database = types.ModuleType('dataset.database')
    dataset.database.get_object_center = _lookup('object_center')
    dataset.database.get_diameter = _lookup('diameter')
    dataset.database.get_object_vert = _lookup('object_vert')
    sys.modules['dataset'], sys.modules['dataset.database'] = dataset, dataset.database

    from gen6d_b200.database import SyntheticObjectDatabase, ReferenceDatabaseAdapter
    from gen6d_b200 import geometry as G
    syn = SyntheticObjectDatabase(**ref['synthetic_args'])

    class RefDB:                                  # the BaseDatabase interface of a reference CustomDatabase
        def __init__(self, s):
            self.database_name = ref['database_name']
            self.s, self.center, self.object_point_cloud = s, s.center, s.object_point_cloud
            self.poses, self.Ks, self.img_ids = s.poses, s.Ks, s.img_ids
        def get_image(self, img_id):
            return self.s.get_image(img_id)
        def get_K(self, img_id):
            return self.Ks[img_id].copy()
        def get_pose(self, img_id):
            return self.poses[img_id].copy()
        def get_img_ids(self):
            return self.img_ids.copy()

    rdb = RefDB(syn)
    assert not hasattr(rdb, 'object_center')
    refiner = ours.name2network['refiner']({})
    refiner.load_ref_imgs(rdb, rdb.get_img_ids())                    # no adapter in user code
    assert isinstance(refiner.ref_database, ReferenceDatabaseAdapter)
    np.testing.assert_allclose(refiner.ref_database.object_center(), ref['object_center'])
    assert refiner.ref_database.object_diameter() == ref['diameter']
    np.testing.assert_allclose(refiner.ref_database.object_vert(), ref['object_vert'])
    q = rdb.get_img_ids()[5]
    a = G.refine_problem(refiner.ref_database, refiner.ref_ids, rdb.get_image(q), rdb.get_K(q), rdb.get_pose(q), 128, 6, True, warp=True)
    b = G.refine_problem(syn, syn.get_img_ids(), syn.get_image(q), syn.get_K(q), syn.get_pose(q), 128, 6, True, warp=True)
    for k in ('que_img', 'que_K', 'que_pose', 'ref_imgs', 'ref_Ks', 'ref_poses'):
        np.testing.assert_array_equal(a[k], b[k])
    # the reference's ref_info keys are a subset of ours + 'masks' (estimator.py:168; masks are unused downstream)
    print('reference database through load_ref_imgs / refine_problem ok')
''')


def test_reference_estimator_binds_this_package():
    r = subprocess.run([sys.executable, '-c', SCRIPT % {'root': ROOT}], capture_output=True, text=True, timeout=300,
                       cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert 'signatures ok' in r.stdout and 'estimator calls bind' in r.stdout
    assert 'load_ref_imgs / refine_problem ok' in r.stdout
