"""Golden vectors of video tracking, produced by the UNMODIFIED reference on CPU: its estimator run with predict.py's
loop semantics (predict with refine_iter 3 on frame 0, then refine_iter 1 from the previous pose), and predict.py's
smoothing (utils/base_utils.project_points, predict.weighted_pts, utils/pose_utils.pnp) of the raw poses; plus a
smoothing-only set of random pose histories.  Needs a reference checkout named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_track.py
Outputs tests/golden/track_golden.npz (frame poses, not images: the tests re-render the frames)."""
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
import plot_stubs  # noqa: E402

plot_stubs.install()
import cases  # noqa: E402
import track_cases  # noqa: E402
from dataset.database import CustomDatabase, get_ref_point_cloud  # noqa: E402  (reference)
from estimator import Gen6DEstimator as RefEstimator  # noqa: E402  (reference)
from predict import weighted_pts  # noqa: E402  (reference)
from utils.base_utils import project_points  # noqa: E402  (reference)
from utils.draw_utils import pts_range_to_bbox_pts  # noqa: E402  (reference)
from utils.pose_utils import pnp  # noqa: E402  (reference)

from gen6d_b200.database import SyntheticObjectDatabase  # noqa: E402
from gen6d_b200.network import name2network as ours  # noqa: E402
from gen6d_b200.weights import seeded_state_dict  # noqa: E402

torch.set_num_threads(os.cpu_count())
EST = cases.estimator_case()
syn = SyntheticObjectDatabase(**EST['db'])
E = np.load(os.path.join(HERE, 'est_golden.npz'))
NUM, STD = 5, 2.5             # predict.py --num / --std defaults


class RefDB(CustomDatabase):
    """Reference-side view of the synthetic database (as in make_golden_estimator.py)."""

    def __init__(self, s):
        self.database_name = 'custom/synthetic'
        self.s = s
        self.center = s.center
        self.object_point_cloud = s.object_point_cloud
        self.poses, self.Ks, self.img_ids = s.poses, s.Ks, s.img_ids

    def get_image(self, img_id):
        return self.s.get_image(img_id)


def smooth(bbox, raw_poses, K, num, std):
    """predict.py:61-70 over a sequence of raw poses, through the reference's functions."""
    hist, proj, avg, out = [], [], [], []
    for pose in raw_poses:
        pts, _ = project_points(bbox, pose, K)
        hist.append(pts)
        pts_ = weighted_pts(hist, weight_num=num, std_inv=std)
        proj.append(pts)
        avg.append(pts_)
        out.append(pnp(bbox, pts_, K))
    return np.stack(proj), np.stack(avg), np.stack(out)


out = {}
# ---------------------------------------------------------------- smoothing only
for num in (5, 10):
    for std in (2.5, 4.0):
        for rep in range(2):
            c = track_cases.smoothing_case(seed=1000 + 10 * num + int(std * 2) + 100 * rep)
            bbox = pts_range_to_bbox_pts(np.max(c['pts'], 0), np.min(c['pts'], 0))
            proj, avg, sm = smooth(bbox, c['poses'], c['K'], num, std)
            key = f'smooth.{num}.{std}.{rep}'
            out[key + '.bbox'], out[key + '.K'], out[key + '.poses'] = bbox, c['K'], c['poses']
            out[key + '.proj'], out[key + '.avg'], out[key + '.smoothed'] = proj, avg, sm

# ---------------------------------------------------------------- the tracked sequence
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
object_pts = get_ref_point_cloud(db)
bbox = pts_range_to_bbox_pts(np.max(object_pts, 0), np.min(object_pts, 0))
q_id = str(int(E['est.query_id']))
gt = track_cases.track_case(syn.get_pose(q_id))
K = syn.K
raw, chains = [], []
pose_init = None
for t in range(len(gt)):
    img = syn.render(gt[t], K)
    est.cfg['refine_iter'] = 3 if pose_init is None else 1           # predict.py:56-57
    pose_pr, inter = est.predict(img, K, pose_init=pose_init)
    pose_init = pose_pr
    raw.append(pose_pr)
    chains.append(np.stack(inter['refine_poses'], 0))
    print('frame', t, 'raw pose t', pose_pr[:, 3], 'gt t', gt[t][:, 3])
proj, avg, sm = smooth(bbox, raw, K, NUM, STD)
out['track.query_id'] = np.asarray(int(q_id))
out['track.gt_poses'], out['track.K'], out['track.bbox'] = gt, K, bbox
out['track.raw_poses'] = np.stack(raw, 0)
out['track.chain0'] = chains[0]                                       # [4,3,4]: frame 0's full prediction
out['track.chains'] = np.stack(chains[1:], 0)                         # [T-1,2,3,4]: one refinement per later frame
out['track.proj'], out['track.avg'], out['track.smoothed'] = proj, avg, sm
out['track.num'], out['track.std'] = np.asarray(NUM), np.asarray(STD)
np.savez_compressed(os.path.join(HERE, 'track_golden.npz'), **out)
print('wrote track_golden.npz', sum(v.nbytes for v in out.values()) / 1e6, 'MB raw')
