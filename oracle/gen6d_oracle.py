"""CPU oracle for the Gen6D three-stage inference hot path.

TEST INFRASTRUCTURE ONLY.  This file is a functional, state-dict-driven restatement (torch fp32
on CPU) of what the reference computes on the path SURVEY.md section 8 scopes.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may import
it, and only as the checker / the timed CPU baseline -- never as part of the shipped GPU path
(gen6d_b200/ never imports oracle/).

Parity pinning: the reference ships no tests or golden vectors for this path (SURVEY.md 4,
8c), so the oracle is pinned against outputs of the UNMODIFIED reference imported in the build
container: tests/golden/make_golden.py runs /root/reference on seeded weights + inputs and
commits the results under tests/golden/; tests/test_oracle_golden.py checks every function
below against those vectors.  Arithmetic lives in torch 2.11 ATen CPU kernels on both sides.

Every function cites the reference file:line it restates.  All tensors are fp32, NCHW, CPU.
`sd` is always a reference-format state dict (the `network_state_dict` of a checkpoint).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)

# torchvision vgg11_bn 'A' feature stack as cut by the reference (network/pretrain_models.py:86-111):
# conv indices grouped by resolution block; BN sits at conv+1, ReLU at conv+2, a 2x2 max-pool
# opens every block but the first.
_VGG_BLOCKS = ((0,), (4,), (8, 11), (15, 18), (22, 25))


def _img_norm(x):
    """torchvision Normalize(mean, std) on NCHW (network/detector.py:156,189)."""
    mean = torch.tensor(IMAGENET_MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


def vgg_pyramid(sd, prefix, x):
    """All block outputs of the VGG11-BN stack (network/pretrain_models.py:17-31,61-72).

    Returns [1/1, 1/2, 1/4, 1/8, 1/16 (PRE-ReLU), 1/32 (max-pool of the pre-ReLU 1/16 map)].
    BN runs in eval mode (running stats); the last conv of the 1/16 block has BN but no ReLU
    because the reference slices features[21:27] (index 27, the ReLU, is excluded).
    """
    outs = []
    for bi, convs in enumerate(_VGG_BLOCKS):
        if bi > 0:
            x = F.max_pool2d(x, 2, 2)
        for ci in convs:
            f = f'{prefix}features.'
            x = F.conv2d(x, sd[f'{f}{ci}.weight'], sd[f'{f}{ci}.bias'], padding=1)
            x = F.batch_norm(x, sd[f'{f}{ci + 1}.running_mean'], sd[f'{f}{ci + 1}.running_var'],
                             sd[f'{f}{ci + 1}.weight'], sd[f'{f}{ci + 1}.bias'], training=False, eps=1e-5)
            if ci != 25:
                x = F.relu(x)
        outs.append(x)
    outs.append(F.max_pool2d(x, 2, 2))
    return outs


def vgg_v1(sd, prefix, x):
    """VGGBNPretrain.forward -> (1/8, 1/16 pre-ReLU, 1/32) (pretrain_models.py:17-31)."""
    p = vgg_pyramid(sd, prefix, x)
    return p[3], p[4], p[5]


def vgg_v3(sd, prefix, x):
    """VGGBNPretrainV3.forward -> (1/4, 1/8, 1/16 pre-ReLU) (pretrain_models.py:61-72)."""
    p = vgg_pyramid(sd, prefix, x)
    return p[2], p[3], p[4]


# ----------------------------------------------------------------------------------------------
# Detector (network/detector.py)
# ----------------------------------------------------------------------------------------------
DET_DEFAULT_CFG = {
    'vgg_score_stats': [[36.264317, 13.151907], [13910.291, 5345.965], [829.70807, 387.98788]],
    'vgg_score_max': 10,
    'detection_scales': [-1.0, -0.5, 0.0, 0.5],
}


def det_extract(sd, imgs):
    """Detector.extract_feats (detector.py:188-197): normalise + VGG, raw (un-normalised) feats."""
    return vgg_v1(sd, 'backbone.', _img_norm(imgs))


def det_load_refs(sd, ref_imgs):
    """Detector.load_impl (detector.py:199-205): NEAREST resize to 120x120 then features.
    ref_imgs: [rfn,3,128,128] in [0,1].  Returns the three reference feature stacks."""
    ref_imgs = F.interpolate(ref_imgs, size=(120, 120))
    return det_extract(sd, ref_imgs)


def det_raw_correlation(que_feats, ref_feats):
    """The three F.conv2d calls of Detector.get_scores (detector.py:222-224): the query feature
    map cross-correlated with each reference's feature map used as a kernel (zero pad k//2)."""
    out = []
    for q, r in zip(que_feats, ref_feats):
        out.append(F.conv2d(q, r, padding=r.shape[-1] // 2))
    return out  # level 0, 1, 2: [qn, rfn, H/8.., W/8..]


def det_fuse_scores(sd, cfg, raw_scales, hs, ws):
    """The post-correlation part of Detector.detect_impl (detector.py:207-216,225-226,243-247).
    raw_scales[s] = the three raw correlation maps [qn, rfn, H/2^l, W/2^l] of scale s: level l is
    nearest-upsampled by 2^l, normalised and clipped, resized bilinearly to (hs, ws); the scales are
    stacked, run through score_conv and maxed over the references.
    -> (feats [qn, 64, hs, ws], stacked [qn, 3*scales, rfn, hs, ws])."""
    stats, mx = cfg['vgg_score_stats'], cfg['vgg_score_max']
    per_scale = []
    for s0, s1, s2 in raw_scales:
        s2 = F.interpolate(s2, scale_factor=4)
        s1 = F.interpolate(s1, scale_factor=2)
        lv = [torch.clip((s - mu) / sigma, min=-mx, max=mx) for s, (mu, sigma) in zip((s0, s1, s2), stats)]
        sc = torch.stack(lv, 1)  # qn,3,rfn,h,w
        qn, _, rfn, hc, wc = sc.shape
        per_scale.append(F.interpolate(sc.reshape(qn, 3 * rfn, hc, wc), size=(hs, ws), mode='bilinear')
                         .reshape(qn, 3, rfn, hs, ws))
    stacked = torch.cat(per_scale, 1)  # qn, 3*scales, rfn, hs, ws
    x = _seq_conv(sd, 'score_conv', (0, 2), stacked, F.conv3d)
    return torch.max(x, 2)[0], stacked


def det_scale_sizes(hq, wq, scales):
    """Target sizes of the query pyramid (detector.py:236-239): round, then round UP to /32."""
    out = []
    for s in scales:
        ht, wt = int(np.round(hq * 2 ** s)), int(np.round(wq * 2 ** s))
        if ht % 32 != 0:
            ht = (ht // 32 + 1) * 32
        if wt % 32 != 0:
            wt = (wt // 32 + 1) * 32
        out.append((ht, wt))
    return out


def _seq_conv(sd, prefix, idxs, x, conv, relu_between=True, **kw):
    for n, i in enumerate(idxs):
        x = conv(x, sd[f'{prefix}.{i}.weight'], sd[f'{prefix}.{i}.bias'], **kw)
        if relu_between and n + 1 < len(idxs):
            x = F.relu(x)
    return x


def det_detect(sd, cfg, que_imgs, ref_feats, return_taps=False):
    """Detector.detect_impl (detector.py:232-266).  que_imgs [qn,3,h,w] in [0,1]."""
    cfg = {**DET_DEFAULT_CFG, **cfg}
    qn, _, hq, wq = que_imgs.shape
    hs, ws = hq // 8, wq // 8
    raw = [det_raw_correlation(det_extract(sd, F.interpolate(que_imgs, size=(ht, wt), mode='bilinear')), ref_feats)
           for ht, wt in det_scale_sizes(hq, wq, cfg['detection_scales'])]
    feats, stacked = det_fuse_scores(sd, cfg, raw, hs, ws)
    scores = _seq_conv(sd, 'score_predict', (0, 2, 4), feats, F.conv2d, padding=1)
    offset = _seq_conv(sd, 'offset_predict', (0, 2, 4), feats, F.conv2d, padding=1)
    scale = _seq_conv(sd, 'scale_predict', (0, 2, 4), feats, F.conv2d, padding=1)
    out = {'scores': scores, 'select_pr_offset': offset, 'select_pr_scale': scale, 'pool_ratio': 8}
    if return_taps:
        out['stacked'] = stacked
        out['scores_feats'] = feats
    return out


def det_parse(scores, scales, offsets, pool_ratio=8):
    """BaseDetector.parse_detection / get_select_index (detector.py:85-121): first-max flat argmax,
    position = ((x,y) + offset + 0.5)*pool - 0.5, scale = 2**scale."""
    qn, _, hq, wq = scores.shape
    idx = torch.argmax(scores.flatten(1), 1)
    ys, xs = idx // wq, idx % wq
    ar = torch.arange(qn, device=scores.device)
    pos = torch.stack([xs, ys], -1) + offsets[ar, :, ys, xs]
    pos = (pos + 0.5) * pool_ratio - 0.5
    return pos, 2 ** scales[ar, 0, ys, xs], idx


# ----------------------------------------------------------------------------------------------
# Selector (network/selector.py, network/attention.py)
# ----------------------------------------------------------------------------------------------
def sel_feats(sd, imgs):
    """ViewpointSelector.get_feats (selector.py:113-119): VGG + per-pixel L2 normalisation."""
    return [F.normalize(f, dim=1) for f in vgg_v1(sd, 'backbone.', _img_norm(imgs))]


def _mlp_linear(sd, prefix, idxs, x):
    for n, i in enumerate(idxs):
        x = F.linear(x, sd[f'{prefix}.{i}.weight'], sd[f'{prefix}.{i}.bias'])
        if n + 1 < len(idxs):
            x = F.relu(x)
    return x


def sel_viewpoints(ref_poses, object_center, object_vert):
    """Normalised viewpoint directions (selector.py:131-147): camera centres relative to the
    object, expressed in the (x, y, vert) frame anchored on the FIRST reference."""
    cam = -ref_poses[:, :3, :3].permute(0, 2, 1) @ ref_poses[:, :3, 3:]
    cam = cam[..., 0] - object_center[None]
    fwd = cam[0]
    y = torch.linalg.cross(object_vert, fwd)
    x = torch.linalg.cross(y, object_vert)
    R = torch.stack([F.normalize(x, dim=0), F.normalize(y, dim=0), F.normalize(object_vert, dim=0)], 0)
    return F.normalize(cam @ R.T, dim=1)


def sel_load_refs(sd, ref_imgs, ref_poses, object_center, object_vert):
    """ViewpointSelector.extract_ref_feats (selector.py:121-148).
    ref_imgs [an,rfn,3,h,w] in [0,1].  Returns (feature stacks [an,rfn,f,h,w] x3, pose embed [rfn,512])."""
    an, rfn, _, h, w = ref_imgs.shape
    feats = sel_feats(sd, ref_imgs.reshape(an * rfn, 3, h, w))
    feats = [f.reshape(an, rfn, *f.shape[1:]) for f in feats]
    vp = sel_viewpoints(ref_poses, object_center, object_vert)
    embed = _mlp_linear(sd, 'view_point_encoder', (0, 2, 4), vp)
    return feats, embed


def sel_score_vps(que_feats, ref_feats):
    """The rotated-similarity score of selector.py:183-195, per level: s = sum_f q*r per
    location, score = sum_hw s * (s / max_hw s).  Returns [qn,3,rfn,an]."""
    out = []
    for q, r in zip(que_feats, ref_feats):
        r = r.permute(1, 0, 2, 3, 4)  # rfn,an,f,h,w
        s = torch.einsum('qfhw,rafhw->qrahw', q, r).flatten(3)
        out.append(torch.sum(s * (s / s.max(3, keepdim=True)[0]), 3))
    return torch.stack(out, 1)


_TOWERS = (
    # (conv index, followed-by) in corr_conv_list[l] (selector.py:27-69); 'n' IN, 'r' ReLU, 'p' pool
    ((1, 'nr'), (4, 'np'), (7, 'nr'), (10, 'np'), (13, 'nr'), (16, '')),
    ((1, 'nr'), (4, 'np'), (7, 'nr'), (10, '')),
    ((1, 'nr'), (4, '')),
)


def sel_tower(sd, level, x):
    """corr_conv_list[level] on the correlation volume x [qn,512,S,h,w] (selector.py:27-69)."""
    x = F.instance_norm(x)
    for ci, post in _TOWERS[level]:
        p = f'corr_conv_list.{level}.{ci}'
        x = F.conv3d(x, sd[p + '.weight'], sd[p + '.bias'], padding=(0, 1, 1))
        if 'n' in post:
            x = F.instance_norm(x)
        if 'r' in post:
            x = F.relu(x)
        if 'p' in post:
            x = F.max_pool3d(x, (1, 2, 2), (1, 2, 2))
    return x


def _attention_block(sd, p, x, heads=8):
    """AttentionBlock.forward with skip_connect=False, LayerNorm over channels
    (attention.py:4-17,50-68).  x [b,512,n]."""
    b, f, n = x.shape
    conv = lambda name: F.conv1d(x, sd[f'{p}.{name}.weight'], sd[f'{p}.{name}.bias'])
    q = conv('conv_query').reshape(b, f // heads, heads, n)
    k = conv('conv_key').reshape(b, f // heads, heads, n)
    v = conv('conv_feats').reshape(b, f // heads, heads, n)
    d = q.shape[1]
    prob = torch.softmax(torch.einsum('bdhn,bdhm->bhnm', q, k) / d ** .5, dim=-1)
    o = torch.einsum('bhnm,bdhm->bdhn', prob, v).reshape(b, f, n)
    o = F.conv1d(o, sd[f'{p}.conv_merge.weight'], sd[f'{p}.conv_merge.bias'])
    o = F.layer_norm(o.permute(0, 2, 1), (f,), sd[f'{p}.norm.norm.weight'], sd[f'{p}.norm.norm.bias'], 1e-5)
    return o.permute(0, 2, 1)


def sel_forward(sd, que_imgs, ref_feats, ref_pose_embed, return_taps=False):
    """ViewpointSelector.compute_view_point_feats (selector.py:177-215).
    que_imgs [qn,3,128,128] in [0,1]; ref_feats from sel_load_refs.  -> logits, angles [qn,rfn]."""
    que = sel_feats(sd, que_imgs)
    towers = []
    for lvl, (q, r) in enumerate(zip(que, ref_feats)):
        r = r.permute(1, 0, 2, 3, 4)
        corr = q[:, None, None] * r[None]  # qn,rfn,an,f,h,w
        qn, rfn, an, f, h, w = corr.shape
        corr = corr.permute(0, 3, 1, 2, 4, 5).reshape(qn, f, rfn * an, h, w)
        t = sel_tower(sd, lvl, corr)
        towers.append(t.reshape(qn, t.shape[1], rfn, an, *t.shape[-2:]))
    vps = sel_score_vps(que, ref_feats)  # qn,3,rfn,an
    x = torch.cat(towers, 1)
    qn, f, rfn, an, h, w = x.shape
    x = x.reshape(qn, f, rfn * an, h, w)
    x = F.conv3d(x, sd['corr_feats_conv.0.weight'], sd['corr_feats_conv.0.bias'])
    x = F.relu(F.instance_norm(x))
    x = F.conv3d(x, sd['corr_feats_conv.3.weight'], sd['corr_feats_conv.3.bias'])
    x = F.avg_pool3d(x, (1, 4, 4))[..., 0, 0].reshape(qn, -1, rfn, an)
    feats = torch.cat([x, F.instance_norm(vps)], 1)  # qn,515,rfn,an
    sp = F.conv2d(F.relu(F.conv2d(feats, sd['score_process.0.weight'], sd['score_process.0.bias'])),
                  sd['score_process.2.weight'], sd['score_process.2.bias'])
    sf = torch.max(sp, 3)[0] + ref_pose_embed.T.unsqueeze(0)  # qn,512,rfn
    for i in range(2):
        msg = _attention_block(sd, f'atts.{i}', sf)
        y = torch.cat([sf, msg], 1)
        y = F.relu(F.instance_norm(F.conv1d(y, sd[f'mlps.{i}.0.weight'], sd[f'mlps.{i}.0.bias'])))
        y = F.relu(F.instance_norm(F.conv1d(y, sd[f'mlps.{i}.3.weight'], sd[f'mlps.{i}.3.bias'])))
        sf = y + sf
    logits = _seq_conv(sd, 'score_predict', (0, 2), sf, F.conv1d)[:, 0]
    af = feats.permute(0, 1, 3, 2).reshape(qn, feats.shape[1] * an, rfn)
    angles = _seq_conv(sd, 'angle_predict', (0, 2, 4), af, F.conv1d)[:, 0]
    if return_taps:
        return logits, angles, {'score_vps': vps, 'towers': towers, 'corr_feats': x, 'scores_feats': sf}
    return logits, angles


def sel_select(logits, angles):
    """select_que_imgs post-processing (selector.py:172-175)."""
    idx = torch.argmax(logits, 1)
    return idx, angles[torch.arange(idx.shape[0], device=idx.device), idx]


# ----------------------------------------------------------------------------------------------
# Refiner (network/refiner.py, network/operator.py)
# ----------------------------------------------------------------------------------------------
def ref_feature_net(sd, imgs):
    """RefineFeatureNet.forward (refiner.py:64-78): [n,3,128,128] -> [n,128,32,32]."""
    p = 'feature_net.'
    x0, x1, x2 = [F.normalize(t, dim=1) for t in vgg_v3(sd, p + 'backbone.', _img_norm(imgs))]

    def block(name, x):
        x = F.conv2d(x, sd[f'{p}{name}.0.weight'], sd[f'{p}{name}.0.bias'], padding=1)
        x = F.relu(F.instance_norm(x))
        x = F.conv2d(x, sd[f'{p}{name}.3.weight'], sd[f'{p}{name}.3.bias'], padding=1)
        return F.instance_norm(x)

    y0 = block('conv0', x0)
    y1 = F.interpolate(block('conv1', x1), scale_factor=2, mode='bilinear')
    y2 = F.interpolate(block('conv2', x2), scale_factor=4, mode='bilinear')
    return block('conv_out', torch.cat([y0, y1, y2], 1))


def ref_sample_volume(feats, verts, projs, h_in, w_in):
    """VolumeRefiner.interpolate_volume_feats + normalize_coords (refiner.py:183-206,
    operator.py:4-17).  feats [b,f,h,w]; verts [b,n,3]; projs [b,3,4] -> [b,f,n]."""
    R, t = projs[:, :3, :3], projs[:, :3, 3:]
    p = verts @ R.permute(0, 2, 1) + t.permute(0, 2, 1)
    depth = p[:, :, 2:].clone()
    depth[depth < 1e-4] = 1e-4
    uv = p[:, :, :2] / depth
    uv = uv + 0.5
    uv = torch.stack([uv[..., 0] / w_in, uv[..., 1] / h_in], -1)
    uv = (uv - 0.5) * 2
    out = F.grid_sample(feats, uv[:, None], mode='bilinear', align_corners=False)  # b,f,1,n
    return out[:, :, 0]


def ref_volume_coords(poses_in, sn):
    """Unit-cube grid rotated by the input pose (refiner.py:211-222): row vectors @ R_in."""
    c = torch.linspace(-1, 1, sn, dtype=torch.float32, device=poses_in.device).to(poses_in.dtype)   # fp32 grid, as the reference
    g = torch.stack(torch.meshgrid(c, c, c, indexing='ij'), -1).reshape(1, sn ** 3, 3)
    return g @ poses_in[:, :3, :3]  # qn, sn^3, 3


def ref_build_volume(sd, que_imgs, que_Ks, que_poses, ref_imgs, ref_Ks, ref_poses, sn):
    """VolumeRefiner.construct_feature_volume (refiner.py:208-247).
    -> mean, std (unbiased, over the refs), in  each [qn,128,sn,sn,sn]."""
    qn = que_imgs.shape[0]
    coords = ref_volume_coords(que_poses, sn)
    ref_proj = ref_Ks @ ref_poses
    h_in, w_in = ref_imgs.shape[-2:]
    means, stds = [], []
    for qi in range(qn):
        rf = ref_feature_net(sd, ref_imgs[qi])
        rfn = rf.shape[0]
        v = ref_sample_volume(rf, coords[qi:qi + 1].repeat(rfn, 1, 1), ref_proj[qi], h_in, w_in)
        means.append(torch.mean(v, 0))
        stds.append(torch.std(v, 0))
    qf = ref_feature_net(sd, que_imgs)
    h_in, w_in = que_imgs.shape[-2:]
    vin = ref_sample_volume(qf, coords, que_Ks @ que_poses, h_in, w_in)
    shp = (qn, -1, sn, sn, sn)
    return torch.stack(means, 0).reshape(shp), torch.stack(stds, 0).reshape(shp), vin.reshape(shp)


def ref_volume_net(sd, mean_in, std):
    """RefineVolumeEncodingNet.forward (refiner.py:88-143); mean_in = cat[mean, in] (256 ch)."""
    p = 'volume_net.'

    def c3(name, x, stride=1):
        return F.conv3d(x, sd[f'{p}{name}.weight'], sd[f'{p}{name}.bias'], stride=stride, padding=1)

    def embed(name, x):
        return c3(f'{name}.3', F.relu(F.instance_norm(c3(f'{name}.0', x))))

    x = torch.cat([embed('mean_embed', mean_in), embed('var_embed', std)], 1)
    for name, stride in (('conv0', 1), ('conv1', 2), ('conv2', 1), ('conv3', 2), ('conv4', 1), ('conv5', 2)):
        x = F.relu(F.instance_norm(c3(f'{name}.0', x, stride)))
    return c3('conv5.3', x)


def ref_regress(sd, x):
    """RefineRegressor.forward (refiner.py:153-166)."""
    p = 'regressor.'
    x = F.leaky_relu(F.linear(x, sd[p + 'fc.0.0.weight'], sd[p + 'fc.0.0.bias']), 0.1)
    x = F.leaky_relu(F.linear(x, sd[p + 'fc.1.0.weight'], sd[p + 'fc.1.0.bias']), 0.1)
    r = F.normalize(F.linear(x, sd[p + 'fcr.weight'], sd[p + 'fcr.bias']), dim=1)
    t = F.linear(x, sd[p + 'fct.weight'], sd[p + 'fct.bias'])
    s = F.linear(x, sd[p + 'fcs.weight'], sd[p + 'fcs.bias'])
    return r, t, s


def ref_forward(sd, que_imgs, que_Ks, que_poses, ref_imgs, ref_Ks, ref_poses, sn=32, return_taps=False):
    """VolumeRefiner.forward in inference mode (refiner.py:249-269).
    que_imgs [qn,3,h,w], que_Ks [qn,3,3], que_poses [qn,3,4], ref_* with an extra rfn axis."""
    mean, std, vin = ref_build_volume(sd, que_imgs, que_Ks, que_poses, ref_imgs, ref_Ks, ref_poses, sn)
    x = ref_volume_net(sd, torch.cat([mean, vin], 1), std)
    r, t, s = ref_regress(sd, x.flatten(1))
    out = {'rotation': r, 'offset': t, 'scale': s}
    if return_taps:
        out.update(mean=mean, std=std, vin=vin, encoded=x)
    return out
