"""Detector on the sm_90a kernels.  Mirrors network/detector.py of the reference: same class
name, cfg keys, checkpoint keys and method contracts (load_ref_imgs / detect_que_imgs numpy API,
load_impl / detect_impl / forward tensor API)."""
from dataclasses import dataclass

import numpy as np
import torch

from .. import ops
from .backbone import pack_vgg, vgg_v1
from .base import Branches, PackedModule
from .params import VGG11BNParams, detector_heads


@dataclass
class DetectorRefs:
    """One object's reference state of the detector (detector.py:199-205)."""
    center_feats: list      # 3 x [rfn, k, k, 512] channels-last (reference keeps NCHW)
    kernels: list           # the same features packed as correlation kernels (Detector.pack_kernels)
    shape: tuple = (120, 120)

    @property
    def rfn(self):
        return self.center_feats[0].shape[0]


class Detector(PackedModule):
    default_cfg = {
        'vgg_score_stats': [[36.264317, 13.151907], [13910.291, 5345.965], [829.70807, 387.98788]],
        'vgg_score_max': 10,
        'detection_scales': [-1.0, -0.5, 0.0, 0.5],
        'train_feats': False,
    }

    def __init__(self, cfg):
        self.cfg = {**self.default_cfg, **cfg}
        super().__init__()
        self.backbone = VGG11BNParams()
        for name, mod in detector_heads(64, 3 * len(self.cfg['detection_scales'])).items():
            setattr(self, name, mod)
        self.pool_ratio = 8
        self.refs = None               # DetectorRefs of the object load_ref_imgs / load_impl loaded

    ref_center_feats = property(lambda self: None if self.refs is None else self.refs.center_feats)
    ref_kernels = property(lambda self: None if self.refs is None else self.refs.kernels)
    ref_shape = property(lambda self: None if self.refs is None else list(self.refs.shape))

    # ------------------------------------------------------------------ weights
    def _pack(self):
        p = {'vgg': pack_vgg(self.backbone)}
        sc = self.score_conv
        p['w1'] = sc[0].weight.reshape(64, -1).float().contiguous()
        p['b1'] = sc[0].bias.float().contiguous()
        p['w2'] = sc[2].weight.reshape(64, 64).float().contiguous()
        p['b2'] = sc[2].bias.float().contiguous()
        for head in ('score_predict', 'scale_predict', 'offset_predict'):
            m = getattr(self, head)
            p[head] = [ops.pack_conv(m[i].weight, m[i].bias, pad=1) for i in (0, 2, 4)]
        return p

    # ------------------------------------------------------------------ channels-last cores
    def _features(self, imgs01):
        """imgs01 [n,h,w,3] in [0,1] -> VGG features (detector.py:188-197)."""
        return vgg_v1(self.packed()['vgg'], ops.imagenet_norm(imgs01, out_c=4))

    def make_refs(self, ref01):
        """detector.py:199-205: nearest resize to 120x120, features, packed as kernels -> DetectorRefs (not stored)."""
        ref01 = ops.resize_nearest(ref01, 120, 120)
        feats = self._features(ref01)
        return DetectorRefs(feats, self.pack_kernels([feats]), (120, 120))

    def _load_nhwc(self, ref01):
        self.refs = self.make_refs(ref01)
        self.bump_generation()          # captured graphs / worker clones hold pointers to the previous reference set

    def pack_kernels(self, feats_objs):
        """The correlation kernels of one or more objects: feats_objs[o] = 3 x [rfn, k, k, c] (equal shapes over the
        objects).  Per level ONE PackedConv whose output channels are the objects' kernels concatenated, object-major."""
        kernels = []
        for fs in zip(*feats_objs):
            rfn, k, _, c = fs[0].shape
            n_obj = len(fs)
            cat = lambda flats: flats[0] if n_obj == 1 else torch.cat(flats, 0)
            kind = ops.tc_kind_for(c)
            if rfn >= 16 and rfn % 4 == 0 and kind is not None and ops.conv_path() == 'tc' and self.cfg.get('corr_rows', True):
                # Tensor-core path, row-decomposed: the k x k kernels become a 1 x k convolution with
                # k*rfn output channels (channel = ky*rfn + r) whose per-row results g6d_det_corr_rowsum
                # adds up.  N = k*rfn (480 at 15 x 15 x 32 refs) fills full 128-wide MMA tiles; the direct
                # form's N = rfn = 32 pays 40 cycles per MMA against a 16-cycle tensor floor.
                flat = cat([f.permute(1, 0, 2, 3).reshape(k * rfn, k * c).contiguous() for f in fs])   # [(obj, ky, r), (kx, c)], K-major B operand
                pc = ops.PackedConv(None, None, c, n_obj * k * rfn, (1, 1, k), 1, (0, k // 2, k // 2))
                pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, kind)
                pc.rows = (k, rfn)
                pc.max_chain_k = 640        # post-ReLU features x post-ReLU features: same-sign products
            else:
                flat = cat([f.reshape(rfn, k * k * c) for f in fs])
                pc = ops.PackedConv(ops.transpose_to_packed(flat), None, c, n_obj * rfn, (1, k, k), 1, (0, k // 2, k // 2))
                if rfn >= 16 and kind is not None:   # channels-last features [rfn, (ky,kx,c)] are already the K-major B operand
                    pc.w_hi, pc.w_lo, pc.kind = ops.split_operand(flat, kind)
                    pc.max_chain_k = 640
            kernels.append(pc)
        return kernels

    def scale_sizes(self, hq, wq):
        """detector.py:236-239: round(h * 2**s), rounded UP to a multiple of 32."""
        out = []
        for s in self.cfg['detection_scales']:
            ht, wt = int(np.round(hq * 2 ** s)), int(np.round(wq * 2 ** s))
            if ht % 32 != 0:
                ht = (ht // 32 + 1) * 32
            if wt % 32 != 0:
                wt = (wt // 32 + 1) * 32
            out.append((ht, wt))
        return out

    def _raw_correlation(self, que01, kernels=None):
        """The three sliding inner products of detector.py:222-224 for one scale (kernels: another object's
        DetectorRefs.kernels; default the loaded object's)."""
        feats = self._features(que01)
        out = []
        for f, pc in zip(feats, kernels or self.ref_kernels):
            y = ops.conv(f, pc, reuse_im2col=True, fold_splits=True)      # persistent kernel, TMA im2col A, the A-reuse kernel's K order
            rows = getattr(pc, 'rows', None)
            out.append(ops.det_corr_rowsum(y, *rows) if rows is not None else y)
        return out

    def _raw_correlation_objects(self, que01, kernels, n_obj, rfn):
        """_raw_correlation for n_obj objects (pack_kernels of their features): the query's features once, ONE
        correlation GEMM per level over all objects -> per level the object-major maps [n_obj * qn, H, W, rfn]."""
        feats = self._features(que01)
        out = []
        for f, pc in zip(feats, kernels):
            y = ops.conv(f, pc, reuse_im2col=True, fold_splits=True)
            k = pc.rows[0] if pc.rows is not None else 1
            m = ops.det_corr_rowsum_objects(y, n_obj, k, rfn)
            out.append(m.reshape(n_obj * m.shape[1], *m.shape[2:]))
        return out

    def _detect_nhwc(self, que01, return_taps=False):
        """detector.py:232-266 on [qn,h,w,3] in [0,1].  Returns channels-last maps."""
        if self.ref_kernels is None:
            raise RuntimeError('Detector: load_ref_imgs / load_impl must be called first')
        return self._detect_maps(que01, self._raw_correlation, que01.shape[0], self.refs.rfn, return_taps)

    def _detect_objects_nhwc(self, que01, kernels, n_obj, rfn, return_taps=False):
        """_detect_nhwc for n_obj objects sharing the query pyramid: maps of n_obj * qn rows, object-major."""
        return self._detect_maps(que01, lambda cur: self._raw_correlation_objects(cur, kernels, n_obj, rfn),
                                 n_obj * que01.shape[0], rfn, return_taps)

    def _detect_maps(self, que01, correlate, rows, rfn, return_taps):
        """Scale pyramid (correlate(scaled query) -> 3 raw maps of `rows` rows), fused score_conv and the three heads."""
        p = self.packed()
        qn, hq, wq, _ = que01.shape
        hs, ws = hq // 8, wq // 8
        scales = self.scale_sizes(hq, wq)
        br = Branches(len(scales))          # the scales are independent until the fused head

        def one_scale(ht, wt):
            cur = que01 if (ht, wt) == (hq, wq) else ops.resize_bilinear(que01, ht, wt)
            return correlate(cur)

        maps = [br.run(i, lambda ht=ht, wt=wt: one_scale(ht, wt)) for i, (ht, wt) in enumerate(scales)]
        br.join()
        sizes = [[(r.shape[1], r.shape[2]) for r in raw] for raw in maps]
        feats = ops.det_score_fuse(maps, sizes, rfn, hs, ws, self.cfg['vgg_score_stats'], self.cfg['vgg_score_max'],
                                   p['w1'], p['b1'], p['w2'], p['b2'], rows)
        outs = {}
        heads = ('score_predict', 'scale_predict', 'offset_predict')
        hb = Branches(len(heads))

        def one_head(head):
            x = feats
            for i, pc in enumerate(p[head]):
                x = ops.conv(x, pc, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE, reuse_im2col=True, fold_splits=True)
            return x

        for i, head in enumerate(heads):
            outs[head] = hb.run(i, lambda head=head: one_head(head))
        hb.join()
        if return_taps:
            outs['raw'] = maps
            outs['scores_feats'] = feats
        return outs

    def _detect_u8(self, u8, refs=None):
        """uint8 frame(s) on the device -> [qn,4] (x, y, scale, score); one capturable stage.  refs: another object's
        DetectorRefs (make_refs_u8) to detect instead of the loaded object; the same launches as a detector loaded with it."""
        que01 = ops.preprocess_u8(u8, out_c=3, imagenet_norm=False)
        if refs is None:
            o = self._detect_nhwc(que01)
        else:
            o = self._detect_maps(que01, lambda cur: self._raw_correlation(cur, refs.kernels), que01.shape[0], refs.rfn, False)
        out, _ = ops.det_parse(o['score_predict'], o['scale_predict'], o['offset_predict'], self.pool_ratio)
        return out

    # ------------------------------------------------------------------ reference tensor API (NCHW)
    def load_impl(self, ref_imgs):
        with torch.no_grad():
            self._load_nhwc(ops.nchw_to_nhwc(ref_imgs.float().contiguous()))

    def detect_impl(self, que_imgs):
        with torch.no_grad():
            o = self._detect_nhwc(ops.nchw_to_nhwc(que_imgs.float().contiguous()))
            scores = ops.nhwc_to_nchw(o['score_predict'])
            offset = ops.nhwc_to_nchw(o['offset_predict'])
            scale = ops.nhwc_to_nchw(o['scale_predict'])
            _, idx = ops.det_parse(o['score_predict'], o['scale_predict'], o['offset_predict'], self.pool_ratio)
        ws = scores.shape[-1]
        que_select_id = torch.stack([idx % ws, idx // ws], 1)
        return {'scores': scores, 'que_select_id': que_select_id, 'pool_ratio': self.pool_ratio,
                'select_pr_offset': offset, 'select_pr_scale': scale}

    def forward(self, data):
        self.load_impl(data['ref_imgs_info']['imgs'])
        return self.detect_impl(data['que_imgs_info']['imgs'])

    # ------------------------------------------------------------------ reference numpy API
    def load_ref_imgs(self, ref_imgs):
        """@param ref_imgs: uint8 [rfn,h,w,3] (detector.py:277-289)"""
        self.refs = self.make_refs_u8(ref_imgs)
        self.bump_generation()          # captured graphs / worker clones hold pointers to the previous reference set

    def make_refs_u8(self, ref_imgs):
        """What load_ref_imgs computes, returned as a DetectorRefs instead of stored."""
        with torch.no_grad():
            u8 = self._to_dev(ref_imgs)
            return self.make_refs(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False))

    def detect_que_imgs(self, que_imgs, que_dev=None):
        """@param que_imgs: uint8 [qn,h,w,3] -> {'positions': f32 [qn,2], 'scales': f32 [qn]} (detector.py:291-304)
        que_dev: the same frames already on the device (upload_frame), to skip the upload."""
        with torch.no_grad():
            out = self.stages.run('detect', self._detect_u8, [self._to_dev(que_imgs) if que_dev is None else que_dev])
            out = self._to_host(out)
        return {'positions': out[:, :2].copy(), 'scales': out[:, 2].copy()}
