"""How sensitive is the UNMODIFIED reference's own detect->select->refine chain to its input?  The
full-chain parity test compares poses after three refinement iterations; with the seeded random
weights every stage amplifies an input difference (each refinement re-crops the images at the previous
pose).  This script measures that amplification on the reference itself (CPU, via ref_shims): the
golden frame's refinement chain from the golden initial pose, and from that pose perturbed by a rotation
of 1e-3 rad and a 1e-3 relative translation -- the size of difference that fp32 summation order in the
detector / selector produces.  tests/test_estimator_gpu.py bounds the GPU path's deviation by the
reference's own gain.  Needs a reference checkout
named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_sensitivity.py
Outputs tests/golden/sens_golden.npz."""
import os
import sys
import tempfile

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import ref_shims  # noqa: E402

ref_shims.install()
import cases  # noqa: E402
from dataset.database import CustomDatabase  # noqa: E402  (reference)
from estimator import Gen6DEstimator as RefEstimator  # noqa: E402  (reference)
from utils import pose_utils as RP  # noqa: E402

from gen6d_b200.database import SyntheticObjectDatabase  # noqa: E402
from gen6d_b200.network import name2network as ours  # noqa: E402
from gen6d_b200.weights import seeded_state_dict  # noqa: E402

torch.set_num_threads(os.cpu_count())
EST = cases.estimator_case()
syn = SyntheticObjectDatabase(**EST['db'])
E = np.load(os.path.join(HERE, 'est_golden.npz'))


class RefDB(CustomDatabase):
    def __init__(self, s):
        self.database_name = 'custom/synthetic'
        self.s, self.center, self.object_point_cloud = s, s.center, s.object_point_cloud
        self.poses, self.Ks, self.img_ids = s.poses, s.Ks, s.img_ids

    def get_image(self, img_id):
        return self.s.get_image(img_id)


db = RefDB(syn)
work = tempfile.mkdtemp(prefix='g6d_ref_')
os.chdir(work)
cfg = {'name': 'gen6d_synth', 'type': 'gen6d', 'ref_resolution': 128, 'ref_view_num': 64, 'det_ref_view_num': 32,
       'refine_iter': 3}
for name, extra in (('detector', {'vgg_score_stats': cases.DET_STATS_EST}), ('selector', {}), ('refiner', {})):
    sub = {'name': f'{name}_synth', 'network': name, **EST['net_cfg'].get(name, {}), **extra}
    os.makedirs(f'data/model/{sub["name"]}', exist_ok=True)
    sd = seeded_state_dict(ours[name](sub), cases.WEIGHT_SEED)
    torch.save({'network_state_dict': sd, 'step': 0}, f'data/model/{sub["name"]}/model_best.pth')
    with open(f'{name}.yaml', 'w') as f:
        yaml.safe_dump(sub, f)
    cfg[name] = f'{name}.yaml'
est = RefEstimator(cfg)
est.build(db, 'all')

q = str(int(E['est.query_id']))
img, K = syn.get_image(q), syn.get_K(q)
P0 = E['est.refine_poses'][0].astype(np.float32)
_, base = est.predict(img, K, pose_init=P0)
base = np.stack(base['refine_poses'], 0)
assert np.abs(base - E['est.refine_poses']).max() < 1e-5, 'the golden chain does not reproduce'
out = {'init': P0, 'base': base}
rng = np.random.RandomState(0)
gains = []
for trial in range(4):
    ax = rng.randn(3)
    ax /= np.linalg.norm(ax)
    ang = 1e-3
    qv = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax])
    P1 = np.concatenate([RP.quat2mat(qv) @ P0[:, :3], P0[:, 3:] * (1 + 1e-3 * rng.randn())], 1).astype(np.float32)
    _, it = est.predict(img, K, pose_init=P1)
    ch = np.stack(it['refine_poses'], 0)
    dR = np.abs(ch[:, :, :3] - base[:, :, :3]).reshape(4, -1).max(1)
    dt = np.abs(ch[:, :, 3] - base[:, :, 3]).max(1) / np.linalg.norm(base[:, :, 3], axis=1)
    print('trial', trial, 'per-iteration max |dR|', dR, 'relative |dt|', dt)
    out[f'pert{trial}'] = ch
    gains.append(np.stack([dR, dt], 0))
g = np.stack(gains, 0)                 # [trial, (R, t), iteration]
out['dR'] = g[:, 0]
out['dt'] = g[:, 1]
out['gain_R'] = (g[:, 0] / g[:, 0, :1]).max(0)         # worst amplification of the rotation difference per iteration
print('worst reference gain of |dR| per iteration:', out['gain_R'])
np.savez_compressed(os.path.join(HERE, 'sens_golden.npz'), **out)
