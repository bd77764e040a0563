"""Golden vectors for BASELINE configs[1]'s detector half at full size, produced by the UNMODIFIED
reference (network/detector.py via ref_shims): 480x640 frame, 32 reference views -> the raw sliding
inner products of detector.py:222-224 (tap D2, BEFORE normalize_scores) for each of the 4 detection
scales and 3 pyramid levels, plus the final maps / argmax.  With rfn = 32 the build routes
the correlation through the tensor-core kernel (network/detector.py: rfn >= 16), which the rfn = 4
case of make_golden.py does not.  Needs a reference checkout
named by GEN6D_REFERENCE, no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden_det32.py
Outputs tests/golden/det32_golden.npz (strided subsamples of the big maps, see `sub`)."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import ref_shims  # noqa: E402

ref_shims.install()
from network import name2network as ref_networks  # noqa: E402  (the reference package)

import cases  # noqa: E402
from gen6d_b200.network import name2network as our_networks  # noqa: E402
from gen6d_b200.weights import seeded_state_dict  # noqa: E402

torch.set_num_threads(os.cpu_count())
out = {}


def sub(t, n=4096):
    f = t.detach().flatten()
    step = max(1, f.numel() // n)
    return f[::step][:n].numpy().copy()


with torch.no_grad():
    c = cases.detector_case_full()
    cfg = {'name': 'det', 'network': 'detector', **c['cfg']}
    det = ref_networks['detector'](cfg)
    det.load_state_dict(seeded_state_dict(our_networks['detector'](cfg), cases.WEIGHT_SEED), strict=True)
    det.eval()
    ref = cases.u8_to_nchw(c['ref_imgs'])
    que = cases.u8_to_nchw(c['que_imgs'])
    det.load_impl(ref)
    qn, _, hq, wq = que.shape
    # the reference's own scale loop (detector.py:236-243), tapping the conv2d of get_scores (:222-224)
    for si, scale in enumerate(det.cfg['detection_scales']):
        ht, wt = int(np.round(hq * 2 ** scale)), int(np.round(wq * 2 ** scale))
        if ht % 32 != 0:
            ht = (ht // 32 + 1) * 32
        if wt % 32 != 0:
            wt = (wt // 32 + 1) * 32
        cur = F.interpolate(que, size=(ht, wt), mode='bilinear') if (ht, wt) != (hq, wq) else que
        qf = det.extract_feats(cur)
        for l, (q, r) in enumerate(zip(qf, det.ref_center_feats)):
            raw = F.conv2d(q, r, padding=r.shape[-1] // 2)
            out[f'raw.s{si}.l{l}.shape'] = np.asarray(raw.shape)
            out[f'raw.s{si}.l{l}.sub'] = sub(raw)
            print(f'scale {si} level {l}: {tuple(raw.shape)} mean {raw.mean():.1f} std {raw.std():.1f}')
    res = det.detect_impl(que)
    out['scores.sub'] = sub(res['scores'])
    out['argmax'] = torch.argmax(res['scores'].flatten(1), 1).numpy()
    top2 = torch.topk(res['scores'].flatten(1), 2, 1)[0]
    out['margin'] = (top2[:, 0] - top2[:, 1]).numpy()
    pos, scl = det.parse_detection(res['scores'], res['select_pr_scale'], res['select_pr_offset'], 8)
    out['positions'], out['scales'] = pos.numpy(), scl.numpy()
    print('argmax', out['argmax'], 'margin', out['margin'], 'positions', out['positions'])

np.savez_compressed(os.path.join(HERE, 'det32_golden.npz'), **out)
print('wrote det32_golden.npz', sum(v.nbytes for v in out.values()) / 1e6, 'MB raw')
