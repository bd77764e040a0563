"""GPU parity of the three networks against the CPU oracle (same seeded weights and inputs) and
against the committed golden vectors of the unmodified reference.  Index selections (detection
cell, viewpoint) must be bit-exact; regressed quantities within the stated fp32 tolerances."""
import os

import numpy as np
import pytest
import torch

from golden import cases
from gen6d_b200.network import name2network
from gen6d_b200.weights import seeded_state_dict
from oracle import gen6d_oracle as O

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'net_golden.npz'))


def close(a, b, rtol=1e-4, atol=1e-4):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def sub(t, n=4096):
    f = t.detach().flatten()
    step = max(1, f.numel() // n)
    return f[::step][:n].cpu().numpy()


def build(name, cfg):
    net = name2network[name](cfg)
    sd = seeded_state_dict(net, cases.WEIGHT_SEED)
    net.load_state_dict(sd, strict=True)
    return net.cuda().eval(), sd


def to_nchw(x):
    return x.permute(0, 3, 1, 2).contiguous().cpu()


# ------------------------------------------------------------------------------------ detector
@pytest.fixture(scope='module')
def det():
    c = cases.detector_case()
    net, sd = build('detector', {'name': 'det', 'network': 'detector', **c['cfg']})
    net.load_ref_imgs(c['ref_imgs'])
    ref_feats = O.det_load_refs(sd, cases.u8_to_nchw(c['ref_imgs']))
    return c, net, sd, ref_feats


def test_detector_reference_features(det):
    c, net, sd, ref_feats = det
    for ours, want in zip(net.ref_center_feats, ref_feats):
        close(to_nchw(ours), want, rtol=1e-4, atol=1e-3)


def test_detector_raw_correlation(det):
    """Tap D2: the sliding inner product before normalisation, vs oracle and golden."""
    from gen6d_b200 import ops
    c, net, sd, ref_feats = det
    que = cases.u8_to_nchw(c['que_imgs'])
    want = O.det_raw_correlation(O.det_extract(sd, que), ref_feats)
    que01 = ops.preprocess_u8(torch.from_numpy(c['que_imgs']).cuda(), out_c=3, imagenet_norm=False)
    got = net._raw_correlation(que01)
    for l, (a, b) in enumerate(zip(got, want)):
        close(to_nchw(a), b, rtol=3e-5, atol=0.5)       # values ~1e5; K = 115200 same-sign terms
        close(to_nchw(a), G[f'det.raw_corr{l}'], rtol=3e-5, atol=0.5)


def test_detector_maps_argmax_positions(det):
    c, net, sd, ref_feats = det
    want = O.det_detect(sd, c['cfg'], cases.u8_to_nchw(c['que_imgs']), ref_feats)
    got = net.detect_impl(cases.u8_to_nchw(c['que_imgs']).cuda())
    close(got['scores'], want['scores'], atol=3e-4)
    close(got['select_pr_offset'], want['select_pr_offset'], atol=3e-4)
    close(got['select_pr_scale'], want['select_pr_scale'], atol=3e-4)
    pos, scl, idx = O.det_parse(want['scores'], want['select_pr_scale'], want['select_pr_offset'])
    top2 = torch.topk(want['scores'].flatten(1), 2, 1)[0]
    print('detector top1-top2 margin (oracle):', (top2[:, 0] - top2[:, 1]).tolist())
    res = net.detect_que_imgs(c['que_imgs'])
    ws = want['scores'].shape[-1]
    sel = got['que_select_id'].cpu()
    assert (sel[:, 1] * ws + sel[:, 0]).tolist() == idx.tolist() == G['det.argmax'].tolist()   # bit-exact cell
    close(res['positions'], pos, atol=2e-2)            # pixels
    close(res['scales'], scl, rtol=2e-3)
    close(res['positions'], G['det.wrap.positions'], atol=2e-2)


def test_detector_tcgen05_correlation_480x640_32refs():
    """BASELINE configs[1], detector half, at full size: 480x640 frame x 32 reference views.  With
    rfn >= 16 the sliding inner product of detector.py:222-224 runs on the tensor-core kernel (refs as the
    K-major B operand, split into short accumulate chains); its raw output per scale and
    level, the final argmax and the decoded position are pinned to the golden run of the unmodified
    reference (tests/golden/make_golden_det32.py)."""
    from gen6d_b200 import ops
    D = np.load(os.path.join(HERE, 'golden', 'det32_golden.npz'))
    c = cases.detector_case_full()
    net, sd = build('detector', {'name': 'det', 'network': 'detector', **c['cfg']})
    net.load_ref_imgs(c['ref_imgs'])
    assert all(k.w_hi is not None for k in net.ref_kernels), 'the tensor-core correlation path is not engaged'
    que01 = ops.preprocess_u8(torch.from_numpy(c['que_imgs']).cuda(), out_c=3, imagenet_norm=False)
    with torch.no_grad():
        o = net._detect_nhwc(que01, return_taps=True)
    worst = 0.0
    for si, per_scale in enumerate(o['raw']):
        for l, raw in enumerate(per_scale):
            got = to_nchw(raw)
            assert list(got.shape) == D[f'raw.s{si}.l{l}.shape'].tolist()
            want = D[f'raw.s{si}.l{l}.sub']
            g = sub(got)
            worst = max(worst, float(np.abs(g - want).max() / np.abs(want).max()))
            close(g, want, rtol=3e-5, atol=0.5)            # values ~1e5; K up to 115200 same-sign terms
    print('raw correlation, worst relative error over 4 scales x 3 levels:', worst, 'reference argmax margin', D['margin'])
    scores = to_nchw(o['score_predict'])
    close(sub(scores), D['scores.sub'], atol=3e-4)
    assert torch.argmax(scores.flatten(1), 1).tolist() == D['argmax'].tolist()          # bit-exact detection cell
    res = net.detect_que_imgs(c['que_imgs'])
    close(res['positions'], D['positions'], atol=2e-2)     # pixels
    close(res['scales'], D['scales'], rtol=2e-3)


# ------------------------------------------------------------------------------------ selector
@pytest.fixture(scope='module')
def sel():
    c = cases.selector_case()
    net, sd = build('selector', {'name': 'sel', 'network': 'selector', **c['cfg']})
    net.load_ref_imgs(c['ref_imgs'], c['ref_poses'], c['object_center'], c['object_vert'])
    feats, embed = O.sel_load_refs(sd, cases.u8_to_nchw(c['ref_imgs']), torch.from_numpy(c['ref_poses']),
                                   torch.from_numpy(c['object_center']), torch.from_numpy(c['object_vert']))
    return c, net, sd, feats, embed


def test_selector_reference_cache(sel):
    c, net, sd, feats, embed = sel
    rfn, an = net.ref_shape
    for ours, want in zip(net.ref_feats_cache, feats):
        h, w, f = ours.shape[1:]
        ours_ = ours.reshape(rfn, an, h, w, f).permute(1, 0, 4, 2, 3)     # -> an,rfn,f,h,w
        close(ours_, want, atol=1e-5)     # L2-normalised VGG features through 8 tensor-core (3xTF32) convs
    close(net.ref_pose_embed, embed, atol=1e-5)


def test_selector_scores_logits_argmax(sel):
    from gen6d_b200 import ops
    c, net, sd, feats, embed = sel
    que = cases.u8_to_nchw(c['que_imgs'])
    logits_w, angles_w, taps = O.sel_forward(sd, que, feats, embed, return_taps=True)
    x = ops.preprocess_u8(torch.from_numpy(c['que_imgs']).cuda(), out_c=4, imagenet_norm=True)
    logits, angles, scores = net._select_nhwc(x)
    rfn, an = net.ref_shape
    close(scores.reshape(-1, 3, rfn, an), taps['score_vps'], rtol=1e-4, atol=1e-5)      # tap S2
    close(scores.reshape(-1, 3, rfn, an), G['sel.score_vps'], rtol=1e-4, atol=1e-5)
    close(logits, logits_w, atol=3e-4)
    close(angles, angles_w, atol=3e-4)
    top2 = torch.topk(logits_w, 2, 1)[0]
    print('selector top1-top2 margin (oracle):', (top2[:, 0] - top2[:, 1]).tolist())
    res = net.select_que_imgs(c['que_imgs'])
    idx, ang = O.sel_select(logits_w, angles_w)
    assert res['ref_idx'].tolist() == idx.tolist() == G['sel.wrap.ref_idx'].tolist()           # bit-exact viewpoint
    close(res['angles'], ang, atol=3e-4)
    close(res['scores'], G['sel.wrap.scores'], atol=3e-4)
    lg2, ang2 = net.compute_view_point_feats(que.cuda())                                      # tensor API
    close(lg2, logits, atol=1e-5)


# ------------------------------------------------------------------------------------ refiner
def test_refiner_volume_and_pose_update():
    c = cases.refiner_case()
    net, sd = build('refiner', {'name': 'ref', 'network': 'refiner'})
    T = torch.from_numpy
    want = O.ref_forward(sd, cases.u8_to_nchw(c['que_imgs']), T(c['que_Ks']), T(c['que_poses']),
                         cases.u8_to_nchw(c['ref_imgs']), T(c['ref_Ks']), T(c['ref_poses']), 32, return_taps=True)
    from gen6d_b200 import ops
    dev = lambda a: T(a).cuda()
    que = ops.preprocess_u8(dev(c['que_imgs']), out_c=4, imagenet_norm=True)
    ref = ops.preprocess_u8(dev(c['ref_imgs']), out_c=4, imagenet_norm=True)
    out, taps = net._forward_nhwc(que, dev(c['que_Ks']), dev(c['que_poses']), ref, dev(c['ref_Ks']),
                                  dev(c['ref_poses']), return_taps=True)
    cl = lambda v: v.permute(0, 4, 1, 2, 3)            # [q,i,j,k,c] -> [q,c,i,j,k]
    mean, vin, std = cl(taps['mean_in'][..., :128]), cl(taps['mean_in'][..., 128:]), cl(taps['std'])
    close(mean, want['mean'], atol=2e-4)               # tap R2
    close(vin, want['vin'], atol=2e-4)
    close(std, want['std'], atol=2e-4)
    close(sub(mean.contiguous(), 16384), G['ref.mean.sub'], atol=2e-4)
    close(out[:, :4], want['rotation'], atol=3e-4)
    close(out[:, 4:6], want['offset'], atol=3e-4)
    close(out[:, 6:7], want['scale'], atol=3e-4)
    close(out[:, :4], G['ref.rotation'], atol=3e-4)
    data = {'que_imgs_info': {'imgs': cases.u8_to_nchw(c['que_imgs']).cuda(), 'Ks_in': dev(c['que_Ks']),
                              'poses_in': dev(c['que_poses'])},
            'ref_imgs_info': {'imgs': cases.u8_to_nchw(c['ref_imgs']).cuda(), 'Ks': dev(c['ref_Ks']),
                              'poses': dev(c['ref_poses'])}, 'inference': True}
    res = net(data)
    close(res['rotation'], out[:, :4], atol=1e-5)
