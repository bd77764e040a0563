"""The synthetic workload used by bench.py, smoke() and the estimator-level tests: seeded
random-weight checkpoints (BASELINE.json: "random weights", no network for pretrained ones), the
procedural object database, and detector score statistics matched to those weights so the
correlation maps are not saturated by the clip (SURVEY.md 8c caution (i))."""
import numpy as np

from .database import SyntheticObjectDatabase
from .network import name2network
from .weights import seeded_state_dict

WEIGHT_SEED = 0
# per-level (mean, std) of the raw detector correlation under WEIGHT_SEED weights
DET_SCORE_STATS = [[106600.0, 29270.0], [68870.0, 23050.0], [18050.0, 5970.0]]
DATABASE = {'n_views': 72, 'height': 480, 'width': 640, 'seed': 7}


def network_cfgs(angle_num=5):
    return {
        'detector': {'name': 'detector_synth', 'network': 'detector', 'vgg_score_stats': DET_SCORE_STATS},
        'selector': {'name': 'selector_synth', 'network': 'selector', 'selector_angle_num': angle_num},
        'refiner': {'name': 'refiner_synth', 'network': 'refiner'},
    }


def seeded_networks(device='cuda', angle_num=5, seed=WEIGHT_SEED):
    nets = {}
    for name, cfg in network_cfgs(angle_num).items():
        net = name2network[name](cfg)
        net.load_state_dict(seeded_state_dict(net, seed), strict=True)
        nets[name] = net.to(device).eval() if device != 'cpu' else net.eval()
    return nets


def seeded_state_dicts(angle_num=5, seed=WEIGHT_SEED):
    return {name: seeded_state_dict(name2network[name](cfg), seed) for name, cfg in network_cfgs(angle_num).items()}


def synthetic_database(**over):
    return SyntheticObjectDatabase(**{**DATABASE, **over})


def build_estimator(database=None, **cfg_over):
    from .estimator import Gen6DEstimator
    est = Gen6DEstimator({'refine_iter': 3, **cfg_over}, modules=seeded_networks())
    database = database or synthetic_database()
    est.build(database, 'all')
    return est, database


def instance_video(copies, T, shift=0.0, depth=1.6, speed=1.5):
    """T frames (480x640) of several objects, several copies each, for multi-instance tracking.  copies: [(database,
    n_copies)]; each copy is its database's view 3 pushed `depth` times further away (about 105x150 px), centred in its
    own cell of a 3x2 grid (at most 6 copies, so no two copies overlap) and moving `speed` px per frame to the right from
    `shift` - 30 px.  Returns (frames, K): K is the first database's view-3 intrinsics, which every copy is rendered with."""
    cells = [(107.0 + 213.0 * (c % 3), 120.0 + 240.0 * (c // 3)) for c in range(6)]
    placed = [db for db, n in copies for _ in range(n)]
    if len(placed) > len(cells):
        raise ValueError(f'instance_video: {len(placed)} copies, at most {len(cells)} fit without overlap')
    db0 = copies[0][0]
    K = db0.get_K(db0.get_img_ids()[3])
    bases = []
    for db in placed:
        pose = db.poses[db.get_img_ids()[3]].copy()
        pose[:, 3] *= depth
        c = K @ (pose[:, :3] @ np.zeros(3) + pose[:, 3])           # the object origin's pixel
        bases.append((db, pose, c[:2] / c[2]))
    frames = []
    for t in range(T):
        img = None
        for (db, pose, (u0, v0)), (cx, cy) in zip(bases, cells):
            p = pose.copy()
            p[0, 3] += (cx - u0 + shift - 30.0 + speed * t) * p[2, 3] / K[0, 0]
            p[1, 3] += (cy - v0) * p[2, 3] / K[1, 1]
            im = db.render(p, K)
            img = im if img is None else np.where((im != db._bg).any(-1, keepdims=True), im, img)
        frames.append(img)
    return frames, K
