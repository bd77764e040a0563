"""Generate the golden vectors under tests/golden/ by running the UNMODIFIED reference
(a liuyuan-pal/Gen6D checkout named by GEN6D_REFERENCE, imported through ref_shims) on the seeded
cases of cases.py.  Needs no GPU:
    GEN6D_REFERENCE=/path/to/Gen6D python tests/golden/make_golden.py
Outputs: net_golden.npz (network-level taps), state_dict_spec.json (checkpoint keys/shapes).
The estimator-level vectors are produced by make_golden_estimator.py.
"""
import json
import os
import sys

import numpy as np
import torch

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
torch.manual_seed(0)
out = {}
spec = {}


def build(name, cfg):
    net = ref_networks[name](cfg)
    sd = seeded_state_dict(our_networks[name](cfg), cases.WEIGHT_SEED)
    net.load_state_dict(sd, strict=True)  # also proves checkpoint-key compatibility
    spec[name] = [[k, list(v.shape), str(v.dtype)] for k, v in net.state_dict().items()]
    return net.eval()


def sub(t, n=4096):
    """Deterministic strided subsample of a big tensor (keeps fixtures small)."""
    f = t.detach().flatten()
    step = max(1, f.numel() // n)
    return f[::step][:n].numpy().copy()


with torch.no_grad():
    # ------------------------------------------------------------------ detector
    c = cases.detector_case()
    det = build('detector', {'name': 'det', 'network': 'detector', **c['cfg']})
    ref = cases.u8_to_nchw(c['ref_imgs'])
    que = cases.u8_to_nchw(c['que_imgs'])
    det.load_impl(ref)
    for l, f in enumerate(det.ref_center_feats):
        out[f'det.ref_feats{l}.sub'] = sub(f)
    # raw correlation at native scale (tap D2, before normalize_scores)
    qf = det.extract_feats(que)
    for l, (q, r) in enumerate(zip(qf, det.ref_center_feats)):
        raw = torch.nn.functional.conv2d(q, r, padding=r.shape[-1] // 2)
        out[f'det.raw_corr{l}'] = raw.numpy()
        print(f'detector raw corr level {l}: mean {raw.mean():.3f} std {raw.std():.3f}')
    res = det.detect_impl(que)
    out['det.scores'] = res['scores'].numpy()
    out['det.offset'] = res['select_pr_offset'].numpy()
    out['det.scale'] = res['select_pr_scale'].numpy()
    pos, scl = det.parse_detection(res['scores'], res['select_pr_scale'], res['select_pr_offset'], 8)
    out['det.positions'] = pos.numpy()
    out['det.scales'] = scl.numpy()
    out['det.argmax'] = torch.argmax(res['scores'].flatten(1), 1).numpy()
    top2 = torch.topk(res['scores'].flatten(1), 2, 1)[0]
    print('detector top1-top2 margin', (top2[:, 0] - top2[:, 1]).tolist(), 'map std', res['scores'].std().item())
    wrap = det.detect_que_imgs(c['que_imgs'])
    out['det.wrap.positions'] = wrap['positions']
    out['det.wrap.scales'] = wrap['scales']

    # ------------------------------------------------------------------ selector
    c = cases.selector_case()
    sel = build('selector', {'name': 'sel', 'network': 'selector', **c['cfg']})
    sel.load_ref_imgs(c['ref_imgs'], c['ref_poses'], c['object_center'], c['object_vert'])
    for l, f in enumerate(sel.ref_feats_cache):
        out[f'sel.ref_feats{l}.sub'] = sub(f)
    out['sel.ref_pose_embed'] = sel.ref_pose_embed.numpy()
    que = cases.u8_to_nchw(c['que_imgs'])
    # score_vps tap (S2): recompute exactly as selector.py:192-194 does
    qf = sel.get_feats(que)
    vps = []
    for q, r in zip(qf, sel.ref_feats_cache):
        r = r.permute(1, 0, 2, 3, 4)
        corr = q[:, None, None] * r[None]
        qn, rfn, an, f, h, w = corr.shape
        corr = corr.permute(0, 3, 1, 2, 4, 5).reshape(qn, f, rfn * an, h, w)
        sm = torch.sum(corr, 1)
        sm_ = sm / (torch.max(sm.flatten(2), 2)[0][..., None, None])
        vps.append(torch.sum(sm.flatten(2) * sm_.flatten(2), 2).reshape(qn, rfn, an))
    out['sel.score_vps'] = torch.stack(vps, 1).numpy()
    logits, angles = sel.compute_view_point_feats(que)
    out['sel.logits'] = logits.numpy()
    out['sel.angles'] = angles.numpy()
    wrap = sel.select_que_imgs(c['que_imgs'])
    out['sel.wrap.ref_idx'] = wrap['ref_idx']
    out['sel.wrap.angles'] = wrap['angles']
    out['sel.wrap.scores'] = wrap['scores']
    top2 = torch.topk(logits, 2, 1)[0]
    print('selector top1-top2 margin', (top2[:, 0] - top2[:, 1]).tolist(), 'logit std', logits.std().item())

    # ------------------------------------------------------------------ refiner
    c = cases.refiner_case()
    rfr = build('refiner', {'name': 'ref', 'network': 'refiner'})
    data = {
        'que_imgs_info': {'imgs': cases.u8_to_nchw(c['que_imgs']), 'Ks_in': torch.from_numpy(c['que_Ks']),
                          'poses_in': torch.from_numpy(c['que_poses'])},
        'ref_imgs_info': {'imgs': cases.u8_to_nchw(c['ref_imgs']), 'Ks': torch.from_numpy(c['ref_Ks']),
                          'poses': torch.from_numpy(c['ref_poses'])},
        'inference': True,
    }
    mean, std, vin, _ = rfr.construct_feature_volume(data['que_imgs_info'], data['ref_imgs_info'],
                                                     rfr.feature_net, 32)
    out['ref.mean.sub'] = sub(mean, 16384)
    out['ref.std.sub'] = sub(std, 16384)
    out['ref.in.sub'] = sub(vin, 16384)
    out['ref.feat_que.sub'] = sub(rfr.feature_net(data['que_imgs_info']['imgs']), 8192)
    res = rfr(data)
    out['ref.rotation'] = res['rotation'].numpy()
    out['ref.offset'] = res['offset'].numpy()
    out['ref.scale'] = res['scale'].numpy()
    print('refiner out', res['rotation'], res['offset'], res['scale'])

np.savez_compressed(os.path.join(HERE, 'net_golden.npz'), **out)
with open(os.path.join(HERE, 'state_dict_spec.json'), 'w') as f:
    json.dump(spec, f)
print('wrote', os.path.join(HERE, 'net_golden.npz'), sum(v.nbytes for v in out.values()) / 1e6, 'MB raw')
