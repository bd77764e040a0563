"""Golden poses + ADD-0.1d / Prj-5 for the north-star acceptance check ("matched ADD-0.1d on
synthetic inputs"), produced by the UNMODIFIED reference: estimator.Gen6DEstimator.build/predict
(CPU, via ref_shims) over N_FRAMES frames of the synthetic object database with the seeded
checkpoints, scored with the reference's utils/pose_utils.py:149-215 (compute_pose_errors /
compute_metrics_impl) against the database's ground-truth poses.  Needs a reference checkout
named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_add.py
Outputs tests/golden/add_golden.npz."""
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
from dataset.database import CustomDatabase, get_diameter  # noqa: E402  (reference)
from estimator import Gen6DEstimator as RefEstimator  # noqa: E402  (reference)
from utils import pose_utils as RP  # noqa: E402

from gen6d_b200.database import SyntheticObjectDatabase  # noqa: E402
from gen6d_b200.network import name2network as ours  # noqa: E402
from gen6d_b200.weights import seeded_state_dict  # noqa: E402

torch.set_num_threads(os.cpu_count())
EST = cases.estimator_case()
syn = SyntheticObjectDatabase(**EST['db'])


class RefDB(CustomDatabase):
    def __init__(self, s):
        self.database_name = 'custom/synthetic'
        self.s = s
        self.center = s.center
        self.object_point_cloud = s.object_point_cloud
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

frame_ids = cases.add_frame_ids(syn)
poses_pr, poses_gt, Ks, det_pos, det_scale, sel_idx, sel_margin, refine = [], [], [], [], [], [], [], []
for fid in frame_ids:
    pose, inter = est.predict(syn.get_image(fid), syn.get_K(fid))
    poses_pr.append(pose.astype(np.float32))
    poses_gt.append(syn.get_pose(fid).astype(np.float32))
    Ks.append(syn.get_K(fid).astype(np.float32))
    det_pos.append(inter['det_position'])
    det_scale.append(inter['det_scale_r2q'])
    sel_idx.append(int(inter['sel_ref_idx']))
    s = np.sort(inter['sel_scores'])
    sel_margin.append(s[-1] - s[-2])
    refine.append(np.stack(inter['refine_poses'], 0))
    print('frame', fid, 'sel', sel_idx[-1], 'margin', sel_margin[-1], 'det scale', det_scale[-1])

pts = syn.object_point_cloud.astype(np.float32)
diameter = float(get_diameter(db))
out = {'frame_ids': np.asarray([int(f) for f in frame_ids]), 'poses_pr': np.stack(poses_pr), 'poses_gt': np.stack(poses_gt),
       'Ks': np.stack(Ks), 'det_position': np.stack(det_pos), 'det_scale': np.asarray(det_scale, np.float32),
       'sel_ref_idx': np.asarray(sel_idx), 'sel_margin': np.asarray(sel_margin, np.float32),
       'refine_poses': np.stack(refine), 'diameter': np.float64(diameter)}
per = [RP.compute_pose_errors(pts, pr, gt, K) for pr, gt, K in zip(poses_pr, poses_gt, Ks)]
out['prj_err'] = np.asarray([p[0] for p in per], np.float64)
out['obj_err'] = np.asarray([p[1] for p in per], np.float64)
res = RP.compute_metrics_impl(pts, diameter, poses_gt, poses_pr, Ks, 1.0, False)
for k, v in res.items():
    out[f'res.{k}'] = np.float64(v)
print('reference metrics', res, 'diameter', diameter)
print('ADD errors / (0.1 d):', (out['obj_err'] / (0.1 * diameter)).round(3))
print('Prj errors (px):', out['prj_err'].round(2))
np.savez_compressed(os.path.join(HERE, 'add_golden.npz'), **out)
print('wrote add_golden.npz', sum(np.asarray(v).nbytes for v in out.values()) / 1e6, 'MB raw')
