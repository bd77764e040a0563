"""Volume refiner on the sm_90a kernels.  Mirrors network/refiner.py of the reference: class
name, cfg keys, checkpoint keys, forward(data) tensor API and the load_ref_imgs /
refine_que_imgs numpy API.

Everything is batched over the qn poses of a call: the 2-D feature net runs once on all
qn*(rfn+1) images, the volume fill on all qn volumes, the 3-D conv stack on [qn, 32,32,32, C];
InstanceNorm groups are per image / per pose, exactly as in the reference (no cross-pose term).
"""
import threading
from dataclasses import dataclass, field

import numpy as np
import torch

from .. import ops
from .backbone import pack_vgg, vgg_v3
from .base import Branches, PackedModule, linear_as_conv
from .params import RefineFeatureParams, RefineRegressorParams, RefineVolumeParams

IN_EPS = 1e-5
_UPLOAD_LOCK = threading.Lock()
# The volume net's and the feature branches' stride-1 convolutions load A by TMA im2col from a split copy of
# their input (prologue applied) on the persistent kernel, in the A-reuse kernel's K order: bit-identical results.
IM2COL = dict(prenorm=True, reuse_im2col=True, fold_splits=True)


@dataclass
class RefinerRefs:
    """One object's reference state of the refiner (refiner.py:271-273): its database, the reference ids, and the
    database images resident on the device (uploaded on first use)."""
    database: object
    ids: list
    dev: dict = field(default_factory=dict)     # image id -> device uint8 [rows, cols, 3]
    src: dict = field(default_factory=dict)     # image id -> geometry.warp_source() of that tensor


class VolumeRefiner(PackedModule):
    default_cfg = {'refiner_sample_num': 32}

    def __init__(self, cfg):
        self.cfg = {**self.default_cfg, **cfg}
        super().__init__()
        self.feature_net = RefineFeatureParams()
        self.volume_net = RefineVolumeParams()
        self.regressor = RefineRegressorParams()
        self.refs = None              # RefinerRefs of the object load_ref_imgs loaded

    ref_database = property(lambda self: None if self.refs is None else self.refs.database)
    ref_ids = property(lambda self: None if self.refs is None else self.refs.ids)

    # ------------------------------------------------------------------ weights
    def _pack(self):
        fn, vn, rg = self.feature_net, self.volume_net, self.regressor
        p = {'vgg': pack_vgg(fn.backbone)}
        for name in fn.BRANCHES:
            m = getattr(fn, name)
            p[name] = (ops.pack_conv(m[0].weight, m[0].bias, pad=1), ops.pack_conv(m[3].weight, m[3].bias, pad=1))
        for name in ('mean_embed', 'var_embed'):
            m = getattr(vn, name)
            p[name] = (ops.pack_conv(m[0].weight, m[0].bias, pad=1), ops.pack_conv(m[3].weight, m[3].bias, pad=1))
        p['trunk'] = []
        for name, _, _, stride in vn.TRUNK:
            m = getattr(vn, name)
            p['trunk'].append(ops.pack_conv(m[0].weight, m[0].bias, stride=stride, pad=1))
        p['conv5_3'] = ops.pack_conv(vn.conv5[3].weight, vn.conv5[3].bias, pad=1)
        # fc.0.0 consumes the flattened [512, 4, 4, 4] volume (channel-major, refiner.py:259); ours is
        # channels-last [4,4,4,512], so permute its input columns once.
        w = rg.fc[0][0].weight
        n_vox = w.shape[1] // 512
        wp = w.reshape(512, 512, n_vox).permute(0, 2, 1).reshape(512, n_vox * 512).float().contiguous()
        p['fc0_w'], p['fc0_b'] = wp, rg.fc[0][0].bias.float().contiguous()
        p['fc0_conv'] = None  # packed lazily for batches > 8 poses
        p['fc1_w'], p['fc1_b'] = rg.fc[1][0].weight.float().contiguous(), rg.fc[1][0].bias.float().contiguous()
        p['fc1_conv'] = None
        p['heads_w'] = torch.cat([rg.fcr.weight, rg.fct.weight, rg.fcs.weight], 0).float().contiguous()
        p['heads_b'] = torch.cat([rg.fcr.bias, rg.fct.bias, rg.fcs.bias], 0).float().contiguous()
        return p

    # ------------------------------------------------------------------ cores (channels-last)
    def _conv_in_conv(self, x, pcs, rows_per_img):
        """conv -> InstanceNorm -> ReLU -> conv -> InstanceNorm (stats returned, not applied)."""
        y, ws = ops.conv(x, pcs[0], stats_rows=rows_per_img, **IM2COL)          # moments fused into the conv epilogue
        ps, pb = ops.instnorm_finalize(ws, rows_per_img, IN_EPS)
        y, ws = ops.conv(y, pcs[1], prologue=ops.PRO_AFFINE_RELU, pro_scale=ps, pro_shift=pb, group_rows=1, stats_rows=rows_per_img,
                         **IM2COL)
        ps, pb = ops.instnorm_finalize(ws, rows_per_img, IN_EPS)
        return y, ps, pb

    def _feature_net(self, imgs_norm4):
        """RefineFeatureNet.forward (refiner.py:64-78): [n,128,128,4] -> [n,32,32,128]."""
        p = self.packed()
        n = imgs_norm4.shape[0]
        x0, x1, x2 = [ops.l2norm_channels(f) for f in vgg_v3(p['vgg'], imgs_norm4)]
        h, w = x0.shape[1], x0.shape[2]
        cat = torch.empty(n, h, w, 192, device=x0.device, dtype=torch.float32)
        br, keep = Branches(3), []

        def one_branch(bi, name, x):
            y, ps, pb = self._conv_in_conv(x, p[name], x.shape[1] * x.shape[2])
            if bi == 0:
                ops.affine_act(y, ps, pb, rows_per_group=h * w, out=cat, out_coff=0)
            else:
                yn = ops.affine_act(y, ps, pb, rows_per_group=y.shape[1] * y.shape[2])
                ops.resize_bilinear(yn, h, w, out=cat, out_coff=64 * bi)   # F.interpolate x2 / x4 bilinear
                keep.append(yn)
            keep.append((y, ps, pb))

        for bi, (name, x) in enumerate((('conv0', x0), ('conv1', x1), ('conv2', x2))):
            br.run(bi, lambda bi=bi, name=name, x=x: one_branch(bi, name, x))
        br.join()
        y, ps, pb = self._conv_in_conv(cat, p['conv_out'], h * w)
        return ops.affine_act(y, ps, pb, rows_per_group=h * w)

    def _volume_net(self, mean_in, stdv):
        """RefineVolumeEncodingNet.forward (refiner.py:88-143) on [qn,sn,sn,sn,C] volumes."""
        p = self.packed()
        qn, sn = mean_in.shape[0], mean_in.shape[1]
        cat = torch.empty(qn, sn, sn, sn, 128, device=mean_in.device, dtype=torch.float32)
        br, keep = Branches(2), []

        def one_embed(bi, name, x):
            y, ws = ops.conv(x, p[name][0], stats_rows=sn ** 3, **IM2COL)
            ps, pb = ops.instnorm_finalize(ws, sn ** 3, IN_EPS)
            ops.conv(y, p[name][1], prologue=ops.PRO_AFFINE_RELU, pro_scale=ps, pro_shift=pb, group_rows=1,
                     out=cat, out_coff=64 * bi, **IM2COL)
            keep.append((y, ps, pb))

        for bi, (name, x) in enumerate((('mean_embed', mean_in), ('var_embed', stdv))):
            br.run(bi, lambda bi=bi, name=name, x=x: one_embed(bi, name, x))
        br.join()
        x, pro, ps, pb = cat, ops.PRO_NONE, None, None
        for pc in p['trunk']:
            vox = ((x.shape[1] - 1) // pc.stride + 1) ** 3                  # output voxels per pose (k 3, pad 1)
            y, ws = ops.conv(x, pc, prologue=pro, pro_scale=ps, pro_shift=pb, group_rows=1, stats_rows=vox, **IM2COL)
            ps, pb = ops.instnorm_finalize(ws, vox, IN_EPS)
            x, pro = y, ops.PRO_AFFINE_RELU
        return ops.conv(x, p['conv5_3'], prologue=pro, pro_scale=ps, pro_shift=pb, group_rows=1, **IM2COL)

    def _regress(self, x):
        """RefineRegressor.forward (refiner.py:153-166); x [qn, n_vox*512] channels-last flattened."""
        p = self.packed()
        qn = x.shape[0]
        if qn <= 8:
            x = ops.linear_smallm(x, p['fc0_w'], p['fc0_b'], act=ops.ACT_LEAKY01)
            x = ops.linear_smallm(x, p['fc1_w'], p['fc1_b'], act=ops.ACT_LEAKY01)
        else:
            if p['fc0_conv'] is None:
                p['fc0_conv'] = linear_as_conv(p['fc0_w'], p['fc0_b'])
                p['fc1_conv'] = linear_as_conv(p['fc1_w'], p['fc1_b'])
            x = ops.conv(x.reshape(qn, 1, 1, -1), p['fc0_conv'], act=ops.ACT_LEAKY01)
            x = ops.conv(x, p['fc1_conv'], act=ops.ACT_LEAKY01).reshape(qn, 512)
        return ops.ref_pose_heads(x, p['heads_w'], p['heads_b'])

    def _forward_nhwc(self, que_norm4, que_Ks, que_poses, ref_norm4, ref_Ks, ref_poses, return_taps=False):
        """que_norm4 [qn,h,w,4]; ref_norm4 [qn,rfn,h,w,4]; Ks/poses as in forward().  -> [qn,7]"""
        qn, rfn, h_in, w_in, _ = ref_norm4.shape
        sn = self.cfg['refiner_sample_num']
        imgs = torch.cat([ref_norm4.reshape(qn * rfn, h_in, w_in, 4), que_norm4], 0)
        feats = self._feature_net(imgs)
        fh, fw, c = feats.shape[1:]
        ref_feats = feats[:qn * rfn].reshape(qn, rfn, fh, fw, c)
        que_feats = feats[qn * rfn:]
        f32 = lambda t: t.to(torch.float32).contiguous()
        mean_in, stdv = ops.ref_volume_fill(ref_feats, que_feats, f32(ref_Ks), f32(ref_poses), f32(que_Ks),
                                            f32(que_poses), sn, h_in, w_in)
        enc = self._volume_net(mean_in, stdv)
        out = self._regress(enc.reshape(qn, -1))
        if return_taps:
            return out, {'mean_in': mean_in, 'std': stdv, 'feats': feats, 'encoded': enc}
        return out

    def _refine_u8(self, que_u8, que_K, que_pose, ref_u8, ref_Ks, ref_poses):
        """uint8 crops + cameras on the device -> [qn,7]; one capturable stage."""
        que = ops.preprocess_u8(que_u8, out_c=4, imagenet_norm=True)
        ref = ops.preprocess_u8(ref_u8, out_c=4, imagenet_norm=True)
        return self._forward_nhwc(que, que_K, que_pose, ref, ref_Ks, ref_poses)

    # ------------------------------------------------------------------ reference tensor API
    def forward(self, data):
        """data['que_imgs_info']: imgs [qn,3,h,w], Ks_in [qn,3,3], poses_in [qn,3,4];
        data['ref_imgs_info']: imgs [qn,rfn,3,h,w], Ks [qn,rfn,3,3], poses [qn,rfn,3,4]
        -> {'rotation' [qn,4], 'offset' [qn,2], 'scale' [qn,1]}  (refiner.py:249-269)."""
        if not data.get('inference', False):
            raise NotImplementedError("inference-only build: pass data['inference'] = True")
        q, r = data['que_imgs_info'], data['ref_imgs_info']
        with torch.no_grad():
            qn, rfn = r['imgs'].shape[:2]
            prep = lambda t: ops.imagenet_norm(ops.nchw_to_nhwc(t.float().contiguous()), out_c=4)
            que = prep(q['imgs'])
            ref = prep(r['imgs'].reshape(qn * rfn, *r['imgs'].shape[2:])).reshape(qn, rfn, *que.shape[1:])
            out = self._forward_nhwc(que, q['Ks_in'], q['poses_in'], ref, r['Ks'], r['poses'])
        return {'rotation': out[:, :4], 'offset': out[:, 4:6], 'scale': out[:, 6:7]}

    # ------------------------------------------------------------------ reference numpy API
    def load_ref_imgs(self, ref_database, ref_ids):
        """refiner.py:271-273.  `ref_database` may be one of this package's ObjectDatabase objects or a
        database of the reference repo (dataset/database.py BaseDatabase), exactly as the reference's
        estimator.py:171 passes it: the latter is wrapped on the fly (the reference reads the object's
        centre / diameter / up vector through free functions, database.py:311-397)."""
        self.refs = self.make_refs(ref_database, ref_ids)
        self.bump_generation()

    @staticmethod
    def make_refs(ref_database, ref_ids):
        """What load_ref_imgs stores, returned as a RefinerRefs (the images are uploaded on first use)."""
        from ..database import as_object_database
        return RefinerRefs(as_object_database(ref_database), ref_ids)

    def _ref_images_dev(self, ids, refs=None):
        """The database images the look-at crops are cut from, resident on the device: all of them
        are uploaded on first use (once per object) and then shared read-only by every worker
        clone / stream, hence the lock and the synchronise before anyone else may see them.
        refs: the RefinerRefs to read (default: the module's own)."""
        refs = self.refs if refs is None else refs
        if not refs.dev:
            with _UPLOAD_LOCK:
                if not refs.dev:
                    dev = {i: torch.from_numpy(np.ascontiguousarray(refs.database.get_image(i))).to(self.device)
                           for i in refs.ids}
                    torch.cuda.current_stream().synchronize()
                    refs.dev.update(dev)
        return [refs.dev[i] for i in ids]

    def _ref_sources(self, ids, refs=None):
        """warp_source() triples of the resident database images `ids` (described once per object)."""
        refs = self.refs if refs is None else refs
        if not refs.src:
            from .. import geometry as G
            dev = self._ref_images_dev(refs.ids, refs)
            refs.src.update({i: G.warp_source(t) for i, t in zip(refs.ids, dev)})
        return [refs.src[i] for i in ids]

    def _refine_warped(self, size):
        """jobs: per pose one query crop followed by its rfn reference crops (qn * (rfn + 1) records)."""
        def fn(jobs, que_K, que_pose, ref_Ks, ref_poses):
            n = jobs.numel() // ops.WARP_JOB_BYTES
            qn = que_K.shape[0]
            crops = ops.warp_perspective_u8(jobs, n, size, size).reshape(qn, n // qn, size, size, 3)
            return self._refine_u8(crops[:, 0].contiguous(), que_K, que_pose, crops[:, 1:].contiguous(), ref_Ks, ref_poses)
        return fn

    def refine_batch(self, frames_dev, que_Ks, in_poses, size=128, ref_num=6, ref_even=False):
        """refine_que_imgs for a batch of independent frames: the host geometry of refiner.py:285-325 per
        frame, then ONE device stage for all of them (look-at crops cut from frames_dev[i] and the resident
        database images, the feature net on qn*(rfn+1) crops, qn volumes, the 3-D stack on [qn,32,32,32,C]),
        one D2H of [qn,7].  Returns the refined poses [qn,3,4] (identical to per-frame refine_que_imgs)."""
        from .. import geometry as G
        qn = len(in_poses)
        probs = G.refine_problems(self.ref_database, self.ref_ids, que_Ks, in_poses, size, ref_num, ref_even)
        srcs, mats = [], []
        for i in range(qn):
            srcs += [G.warp_source(frames_dev[i])] + self._ref_sources(probs['ref_ids'][i])
            mats += [G.perspective_dst_to_src(probs['que_H'][i])] + [G.perspective_dst_to_src(H) for H in probs['ref_Hs'][i]]
        cams = ('que_K', 'que_pose', 'ref_Ks', 'ref_poses')
        with torch.no_grad():
            args = [self._to_dev(G.pack_warp_jobs(srcs, mats))] + [self._to_dev(probs[k]) for k in cams]
            out = self._to_host(self.stages.run(f'refine_warp{size}', self._refine_warped(size), args))
        return G.apply_refinements(probs, out[:, :4], out[:, 4:6], [2.0 ** o[6] for o in out])

    def refine_que_imgs(self, que_img, que_K, in_pose, size=128, ref_num=6, ref_even=False, que_dev=None,
                        host_warps=False):
        """Host wrapper of refiner.py:275-341 (same arguments and result: pose [3,4] float32).
        The look-at crops of the query frame and of the selected reference views are cut on the
        device by g6d_warp_perspective_u8 (bit-exact with cv2.warpPerspective, so the result is the
        same as with host_warps=True, which keeps OpenCV on the host as the reference does).
        que_dev: the frame already on the device (upload_frame), to share it across iterations."""
        from .. import geometry as G
        prob = G.refine_problem(self.ref_database, self.ref_ids, que_img, que_K, in_pose, size, ref_num, ref_even,
                                warp=host_warps)
        cams = ('que_K', 'que_pose', 'ref_Ks', 'ref_poses')
        with torch.no_grad():
            if host_warps:
                args = [self._to_dev(prob[k][None]) for k in ('que_img', 'que_K', 'que_pose', 'ref_imgs', 'ref_Ks', 'ref_poses')]
                out = self.stages.run('refine', self._refine_u8, args)
            else:
                if que_dev is None:
                    que_dev = self.upload_frame(que_img)
                srcs = [que_dev] + self._ref_images_dev(list(prob['ref_ids']))
                mats = [G.perspective_dst_to_src(prob['que_H'])] + [G.perspective_dst_to_src(H) for H in prob['ref_Hs']]
                args = [self._to_dev(G.pack_warp_jobs(srcs, mats))] + [self._to_dev(prob[k][None]) for k in cams]
                out = self.stages.run(f'refine_warp{size}', self._refine_warped(size), args)
            out = self._to_host(out)[0]
        return G.apply_refinement(prob, quat=out[:4], offset=out[4:6], scale=2.0 ** out[6])
