"""Golden vectors for the evaluation metrics (SURVEY §8 row f4) from the UNMODIFIED reference
(utils/pose_utils.py:149-215 compute_pose_errors / compute_metrics_impl).  Needs a reference checkout
named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_metrics.py
Outputs tests/golden/metrics_golden.npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import ref_shims  # noqa: E402

ref_shims.install()
import cases  # noqa: E402
from utils import pose_utils as RP  # noqa: E402  (reference)

c = cases.metrics_case()
out = {}
per_pose = [RP.compute_pose_errors(c['pts'], pr, gt, K) for pr, gt, K in zip(c['pr'], c['gt'], c['Ks'])]
out['prj_err'] = np.asarray([p[0] for p in per_pose], np.float64)
out['obj_err'] = np.asarray([p[1] for p in per_pose], np.float64)
out['pose_err'] = np.asarray([p[2] for p in per_pose], np.float64)
sym = []
for pr, gt in zip(c['pr'], c['gt']):
    a = c['pts'] @ pr[:, :3].T + pr[:, 3][None]
    b = c['pts'] @ gt[:, :3].T + gt[:, 3][None]
    sym.append(np.mean(np.min(np.linalg.norm(a[:, None] - b[None, :], 2, 2), 1)))     # pose_utils.py:194-196
out['obj_err_sym'] = np.asarray(sym, np.float64)
for scale in (1.0, 0.5):
    for symmetric in (False, True):
        res = RP.compute_metrics_impl(c['pts'], c['diameter'], list(c['gt']), list(c['pr']), list(c['Ks']), scale, symmetric)
        for k, v in res.items():
            out[f'res.{scale}.{int(symmetric)}.{k}'] = np.float64(v)
np.savez_compressed(os.path.join(HERE, 'metrics_golden.npz'), **out)
for k, v in out.items():
    print(k, np.asarray(v).round(5) if np.asarray(v).ndim else v)
