"""Generates dropin_golden.json for tests/test_dropin.py from the UNMODIFIED reference (a checkout of
liuyuan-pal/Gen6D named by GEN6D_REFERENCE, imported through ref_shims):

  * signatures: parameter names and default values (repr) of every network method the reference's
    estimator calls, on the reference's own Detector / ViewpointSelector / VolumeRefiner;
  * imports / calls: what estimator.py takes from the `network` package and every call it makes on the
    three networks, constructors included (method, number of positional arguments, keyword names),
    read from its syntax tree;
  * database: the reference's get_object_center / get_diameter / get_object_vert of the seeded
    synthetic object presented as a reference CustomDatabase -- the values estimator.py:171's raw
    database hands to the refiner through those free functions.

    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_dropin.py
"""
import ast
import inspect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), HERE]

import ref_shims  # noqa: E402

NETS = {'detector': 'detector', 'selector': 'selector', 'refiner': 'refiner'}
CALLS = {'detector': ('__init__', 'load_ref_imgs', 'detect_que_imgs', 'forward'),
         'selector': ('__init__', 'load_ref_imgs', 'select_que_imgs', 'forward'),
         'refiner': ('__init__', 'load_ref_imgs', 'refine_que_imgs', 'forward')}
DB_ARGS = dict(n_views=12, height=120, width=160, seed=3)


def default_repr(p):
    return None if p.default is inspect.Parameter.empty else repr(p.default)


def estimator_usage(path):
    tree = ast.parse(open(path).read())
    imports = sorted({a.name for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and n.module == 'network' for a in n.names})
    calls = set()
    for n in ast.walk(tree):
        f = getattr(n, 'func', None)
        if isinstance(n, ast.Call) and isinstance(f, ast.Attribute) and isinstance(f.value, ast.Attribute) \
                and isinstance(f.value.value, ast.Name) and f.value.value.id == 'self' and f.value.attr in NETS:
            calls.add((f.value.attr, f.attr, len(n.args), tuple(sorted(k.arg for k in n.keywords if k.arg))))
        if isinstance(n, ast.Call) and isinstance(f, ast.Subscript) and isinstance(f.value, ast.Name) and f.value.id == 'name2network':
            for net in NETS:                    # name2network[cfg['network']](cfg): any of the three classes
                calls.add((net, '__init__', len(n.args), tuple(sorted(k.arg for k in n.keywords if k.arg))))
    return imports, [list(c[:3]) + [list(c[3])] for c in sorted(calls)]


def main():
    ref_shims.install(networks=True)
    import network as ref_network
    sigs = {f'{name}.{m}': [[p.name, default_repr(p)] for p in inspect.signature(getattr(ref_network.name2network[name], m)).parameters.values()]
            for name, methods in CALLS.items() for m in methods}
    imports, calls = estimator_usage(os.path.join(ref_shims.REFERENCE_ROOT, 'estimator.py'))

    from dataset.database import CustomDatabase, get_diameter, get_object_center, get_object_vert
    from gen6d_b200.database import SyntheticObjectDatabase
    syn = SyntheticObjectDatabase(**DB_ARGS)

    class RefDB(CustomDatabase):
        def __init__(self, s):
            self.database_name = 'custom/synthetic'
            self.s, self.center, self.object_point_cloud = s, s.center, s.object_point_cloud
            self.poses, self.Ks, self.img_ids = s.poses, s.Ks, s.img_ids

        def get_image(self, img_id):
            return self.s.get_image(img_id)

    rdb = RefDB(syn)
    out = {'signatures': sigs, 'estimator_imports': imports, 'estimator_calls': calls,
           'database': {'synthetic_args': DB_ARGS, 'database_name': rdb.database_name,
                        'object_center': [float(v) for v in get_object_center(rdb)],
                        'diameter': float(get_diameter(rdb)),
                        'object_vert': [float(v) for v in get_object_vert(rdb)]}}
    with open(os.path.join(HERE, 'dropin_golden.json'), 'w') as f:
        json.dump(out, f, indent=1)
        f.write('\n')
    print('wrote dropin_golden.json:', len(sigs), 'signatures,', len(calls), 'estimator calls')


if __name__ == '__main__':
    main()
