"""Golden vectors for the host geometry and the full estimator, produced by the UNMODIFIED
reference (estimator.py, utils/*.py, network/*.py via ref_shims) on the synthetic in-memory
object database and the seeded checkpoints.  Needs a reference checkout
named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_estimator.py
Outputs tests/golden/est_golden.npz."""
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
from network.refiner import VolumeRefiner as RefRefiner  # noqa: E402
from utils import base_utils as RB, database_utils as RD, pose_utils as RP  # noqa: E402

from gen6d_b200.database import SyntheticObjectDatabase  # noqa: E402
from gen6d_b200.network import name2network as ours  # noqa: E402
from gen6d_b200.weights import seeded_state_dict  # noqa: E402

torch.set_num_threads(os.cpu_count())
EST = cases.estimator_case()
syn = SyntheticObjectDatabase(**EST['db'])


class RefDB(CustomDatabase):
    """Reference-side view of the synthetic database (isinstance(CustomDatabase) drives the
    reference's get_object_center / get_diameter / get_object_vert dispatch)."""

    def __init__(self, s):
        self.database_name = 'custom/synthetic'
        self.s = s
        self.center = s.center
        self.object_point_cloud = s.object_point_cloud
        self.poses, self.Ks, self.img_ids = s.poses, s.Ks, s.img_ids

    def get_image(self, img_id):
        return self.s.get_image(img_id)


db = RefDB(syn)
out = {}

# ---------------------------------------------------------------- geometry taps
ids = RD.select_reference_img_ids_fps(db, db.get_img_ids(), 64)
out['geo.fps_ids'] = np.asarray([int(i) for i in ids])
imgs, masks, Ks, poses, Hs = RD.normalize_reference_views(db, ids[:6], 128, 0.05)
out['geo.norm.Ks'], out['geo.norm.poses'], out['geo.norm.Hs'] = Ks, poses, Hs
out['geo.norm.imgs'] = imgs[:3]
img0 = db.get_image('3')
crop, M = RB.transformation_crop(img0, np.array([300.5, 260.25], np.float32), 1 / 1.37, 0, 128)
out['geo.crop.img'], out['geo.crop.M'] = crop, M
que_K = syn.K
out['geo.sim_pose'] = RP.estimate_pose_from_similarity_transform_compose(
    np.array([310.0, 225.0], np.float32), np.float32(1.21), np.float32(0.33), poses[2], Ks[2], que_K, db.center)

# refinement host code with the network replaced by fixed outputs
captured = {}
FIXED = {'rotation': torch.tensor([[0.98, 0.05, -0.1, 0.15]]), 'offset': torch.tensor([[1.5, -2.25]]),
         'scale': torch.tensor([[0.12]])}
FIXED['rotation'] = FIXED['rotation'] / FIXED['rotation'].norm()


def fake_forward(self, data):
    captured['que'] = {k: v.numpy().copy() for k, v in data['que_imgs_info'].items()}
    captured['ref'] = {k: v.numpy().copy() for k, v in data['ref_imgs_info'].items()}
    return FIXED


rr = RefRefiner({'name': 'r', 'network': 'refiner'})
rr.load_ref_imgs(db, db.get_img_ids())
orig_forward = RefRefiner.forward
RefRefiner.forward = fake_forward
in_pose = syn.get_pose('5')
in_pose = np.concatenate([RP.quat2mat([0.995, 0.03, -0.05, 0.04]) @ in_pose[:, :3], in_pose[:, 3:] * 1.07], 1).astype(np.float32)
que_img = syn.get_image('5')
pose_out = rr.refine_que_imgs(que_img, que_K, in_pose, size=128, ref_num=6, ref_even=True)
RefRefiner.forward = orig_forward
out['geo.refine.in_pose'] = in_pose
out['geo.refine.que_K'], out['geo.refine.que_pose'] = captured['que']['Ks_in'][0], captured['que']['poses_in'][0]
out['geo.refine.ref_Ks'], out['geo.refine.ref_poses'] = captured['ref']['Ks'][0], captured['ref']['poses'][0]
out['geo.refine.que_img'] = (captured['que']['imgs'][0].transpose(1, 2, 0) * 255).round().astype(np.uint8)
out['geo.refine.ref_img0'] = (captured['ref']['imgs'][0, 0].transpose(1, 2, 0) * 255).round().astype(np.uint8)
out['geo.refine.fixed'] = np.concatenate([FIXED['rotation'][0].numpy(), FIXED['offset'][0].numpy(), FIXED['scale'][0].numpy()])
out['geo.refine.pose_out'] = pose_out

# ---------------------------------------------------------------- full estimator on CPU
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
out['est.ref_imgs0'] = est.ref_info['imgs'][:2]
out['est.ref_poses'] = est.ref_info['poses']
# pick a query frame whose selections are well separated (random weights give random margins;
# parity of index selections is only meaningful when the reference's own margin is not ~0)
refiner_saved, est.refiner = est.refiner, None
q_id = None
for cand in syn.get_img_ids():
    _, it = est.predict(syn.get_image(cand), syn.get_K(cand))
    sc = np.sort(it['sel_scores'])
    print('candidate', cand, 'selector margin', sc[-1] - sc[-2], 'det scale', it['det_scale_r2q'])
    if sc[-1] - sc[-2] > 0.15:
        q_id = cand
        break
est.refiner = refiner_saved
out['est.query_id'] = np.asarray(int(q_id))
pose, inter = est.predict(syn.get_image(q_id), syn.get_K(q_id))
out['est.det_position'], out['est.det_scale'] = inter['det_position'], inter['det_scale_r2q']
out['est.sel_ref_idx'], out['est.sel_angle'] = np.asarray(inter['sel_ref_idx']), np.asarray(inter['sel_angle_r2q'])
out['est.sel_scores'] = inter['sel_scores']
out['est.refine_poses'] = np.stack(inter['refine_poses'], 0)
out['est.pose'] = pose
# tracking mode (predict.py:56-59 style): refinement only, from a perturbed ground-truth pose
gt = syn.get_pose(q_id)
init = np.concatenate([RP.quat2mat([0.997, 0.04, -0.03, 0.05]) @ gt[:, :3], gt[:, 3:] * 1.06], 1).astype(np.float32)
pose_t, inter_t = est.predict(syn.get_image(q_id), syn.get_K(q_id), pose_init=init)
out['est.track_init'] = init
out['est.track_poses'] = np.stack(inter_t['refine_poses'], 0)
print('tracking poses', out['est.track_poses'][-1])
s = np.sort(inter['sel_scores'])
print('estimator: det', inter['det_position'], inter['det_scale_r2q'], 'sel', inter['sel_ref_idx'], inter['sel_angle_r2q'],
      'sel margin', s[-1] - s[-2])
print('pose', pose)
np.savez_compressed(os.path.join(HERE, 'est_golden.npz'), **out)
print('wrote est_golden.npz', sum(v.nbytes for v in out.values()) / 1e6, 'MB raw')
