"""Seeded synthetic inputs shared by the golden-vector generator, the oracle tests and the GPU
parity tests.  Everything is a pure function of the seed (torch CPU generator), so the same
tensors are rebuilt on any machine with this image's torch build; only *outputs* are committed.
"""
import numpy as np
import torch

WEIGHT_SEED = 0

# Detector statistics that keep random-weight correlations inside the +-10 clip window so the
# correlation kernel stays observable in the final maps (SURVEY.md 8c caution (i)).  Measured
# on the seeded checkpoint by make_golden.py (raw per-level mean / std), then frozen here.
DET_STATS = [[106600.0, 29270.0], [68870.0, 23050.0], [18050.0, 5970.0]]


def _g(seed):
    g = torch.Generator(device='cpu')
    g.manual_seed(seed)
    return g


def rand_images_u8(seed, *shape):
    """uint8 images with some spatial structure (blocky low-frequency + noise), NHWC."""
    g = _g(seed)
    *lead, h, w, c = shape
    low = torch.rand(*lead, c, max(h // 16, 1), max(w // 16, 1), generator=g)
    low = torch.nn.functional.interpolate(low.reshape(-1, c, low.shape[-2], low.shape[-1]), size=(h, w),
                                          mode='bilinear', align_corners=False)
    low = low.reshape(*lead, c, h, w)
    noise = torch.rand(*lead, c, h, w, generator=g)
    img = (0.7 * low + 0.3 * noise).clamp(0, 1)
    img = (img * 255).round().to(torch.uint8)
    perm = list(range(len(lead))) + [len(lead) + 1, len(lead) + 2, len(lead)]
    return img.permute(*perm).contiguous().numpy()


def u8_to_nchw(imgs):
    """color_map_forward + NHWC->NCHW (utils/base_utils.py:117-118)."""
    t = torch.from_numpy(imgs.astype(np.float32) / 255)
    nd = t.dim()
    return t.permute(*range(nd - 3), nd - 1, nd - 3, nd - 2).contiguous()


def random_rotation(g):
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))[None]
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


def look_at_pose(cam, up=np.array([0., 0., 1.])):
    """World->camera [R|t] for a camera at `cam` looking at the origin (OpenCV axes: z forward)."""
    z = -cam / np.linalg.norm(cam)
    x = np.cross(z, up)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross(z, np.array([0., 1., 0.]))
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 0)
    return np.concatenate([R, (-R @ cam)[:, None]], 1)


def sphere_poses(seed, n, radius=5.0, jitter=0.0):
    g = _g(seed)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64).numpy()
    d[:, 2] = np.abs(d[:, 2]) * 0.7 + 0.1
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rad = radius * (1 + jitter * (torch.rand(n, generator=g, dtype=torch.float64).numpy() - 0.5))
    return np.stack([look_at_pose(d[i] * rad[i]) for i in range(n)], 0).astype(np.float32)


def detector_case(seed=11, rfn=4, hq=96, wq=128, qn=1):
    return {'ref_imgs': rand_images_u8(seed, rfn, 128, 128, 3),
            'que_imgs': rand_images_u8(seed + 1, qn, hq, wq, 3),
            'cfg': {'vgg_score_stats': DET_STATS}}


def detector_case_full(seed=111):
    """BASELINE configs[1], detector half: 480x640 frame, 32 reference views (the estimator default):
    rfn >= 16 routes the correlation through the tensor-core kernel."""
    return detector_case(seed=seed, rfn=32, hq=480, wq=640)


def selector_case(seed=21, rfn=8, an=5, qn=1):
    poses = sphere_poses(seed + 2, rfn)
    return {'ref_imgs': rand_images_u8(seed, an, rfn, 128, 128, 3),
            'que_imgs': rand_images_u8(seed + 1, qn, 128, 128, 3),
            'ref_poses': poses,
            'object_center': np.zeros(3, np.float32),
            'object_vert': np.array([0, 0, 1], np.float32),
            'cfg': {'selector_angle_num': an}}


def refiner_case(seed=31, qn=2, rfn=6, size=128):
    f = size * 0.95 / 2.0 * 5.0
    K = np.array([[f, 0, size / 2], [0, f, size / 2], [0, 0, 1]], np.float32)
    que_poses = sphere_poses(seed + 2, qn, jitter=0.1)
    ref_poses = np.stack([sphere_poses(seed + 3 + i, rfn, jitter=0.1) for i in range(qn)], 0)
    return {'que_imgs': rand_images_u8(seed, qn, size, size, 3),
            'ref_imgs': rand_images_u8(seed + 1, qn, rfn, size, size, 3),
            'que_Ks': np.repeat(K[None], qn, 0), 'que_poses': que_poses,
            'ref_Ks': np.repeat(K[None, None], qn, 0).repeat(rfn, 1), 'ref_poses': ref_poses}


from gen6d_b200 import synthetic as _syn  # noqa: E402

# Detector statistics for the estimator-level case (480x640 frame of the synthetic object, 32 refs)
DET_STATS_EST = _syn.DET_SCORE_STATS


def estimator_case():
    return {'db': dict(_syn.DATABASE), 'net_cfg': {}, 'query_id': '11'}


def add_frame_ids(db, n=20):
    """The frames of the ADD-0.1d acceptance run: every third view of the synthetic database, n of them."""
    ids = db.get_img_ids()
    return [ids[(3 * i + 1) % len(ids)] for i in range(n)]


def metrics_case(n_pts=700, n_poses=14, seed=77):
    """Seeded inputs of the evaluation metrics (SURVEY §8 row f4): object points on a bumpy ellipsoid,
    ground-truth poses in front of the camera, predictions = ground truth perturbed by amounts that
    straddle the ADD-0.1d and Prj-5 thresholds (plus one pose whose points cross the camera plane)."""
    rng = np.random.RandomState(seed)
    d = rng.randn(n_pts, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = (d * np.array([0.5, 0.8, 1.0]) * (0.8 + 0.2 * rng.rand(n_pts, 1))).astype(np.float32)
    diameter = float(np.max(np.linalg.norm(pts[:, None] - pts[None], axis=2)))

    def rot(v):
        ang = np.linalg.norm(v)
        if ang < 1e-12:
            return np.eye(3)
        k = v / ang
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        return np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx

    gts, prs, Ks = [], [], []
    for i in range(n_poses):
        R = rot(rng.randn(3) * 1.5)
        t = np.array([rng.randn() * 0.3, rng.randn() * 0.3, 4.0 + rng.rand() * 3])
        gt = np.concatenate([R, t[:, None]], 1).astype(np.float32)
        mag = [0.0, 0.002, 0.01, 0.03, 0.06, 0.12, 0.3][i % 7]
        Rp = rot(rng.randn(3) * mag) @ R
        tp = t + rng.randn(3) * mag * np.array([1, 1, 3])
        if i == n_poses - 1:
            tp = np.array([0.05, -0.02, 0.3])          # object straddles the camera plane: exercises the depth clamp
        prs.append(np.concatenate([Rp, tp[:, None]], 1).astype(np.float32))
        gts.append(gt)
        f = 500 + 200 * rng.rand()
        Ks.append(np.array([[f, 0, 320], [0, f, 240], [0, 0, 1]], np.float32))
    return {'pts': pts, 'diameter': diameter, 'gt': np.stack(gts), 'pr': np.stack(prs), 'Ks': np.stack(Ks)}
