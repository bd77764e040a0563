"""Viewpoint selector on the sm_90a kernels.  Mirrors network/selector.py (+ attention.py) of the
reference: class name, cfg keys, checkpoint keys, load_ref_imgs / select_que_imgs numpy API and
extract_ref_feats / compute_view_point_feats / forward tensor API.

Device-side data layout (see DESIGN.md): the cached reference stack is channels-last and
slice-major, ref[l] = [S = rfn*an (r-major, a-minor), h_l, w_l, 512], which is simultaneously
 * the streaming operand of the correlation-score kernel (one 2 KB row per (slice, location)),
 * the input tensor of the first tower convolution, whose loader forms the (never
   materialised) correlation volume q (.) ref with the first InstanceNorm3d folded in.
"""
from dataclasses import dataclass

import numpy as np
import torch

from .. import ops
from .backbone import pack_vgg, vgg_v1
from .base import Branches, PackedModule, linear_as_conv
from .params import SEL_TOWER_POST, SEL_TOWERS, VGG11BNParams, selector_modules

IN_EPS = 1e-5


class LocalComm:
    """Single-process stand-in for gen6d_b200.dist.Comm (no sharding)."""
    rank, world, capturable = 0, 1, True

    def all_reduce_sum(self, t):
        return t

    def all_gather_cat(self, t, dim=0):
        return t

    def shard_range(self, n):
        return 0, n


FEAT_PAD = 516  # 512 correlation features + 3 similarity scores, padded to a multiple of 4
# Queries per batched selection call.  What a chunk holds grows with it: at 64 references x 5 angles a query's
# level-0 16x16 64-channel output is 21 MB, and each batched layer also keeps its input's fp16 hi/lo split copy (the same
# bytes), so the level-0 16x16 layer holds about 63 MB per query, the 8x8 layers about 31 MB and cat_buf 16 MB.  The
# per-query q (.) ref layers' 168 MB split copy of the reference stack is not replicated.  Ten queries fill the waves of
# the 8x8 and 4x4 layers (12.1 of 13 and 6.1 of 7).
SEL_QUERY_CHUNK = 10


@dataclass
class SelectorRefs:
    """One object's reference state of the selector (selector.py:121-148), this rank's shard of it."""
    feats_cache: list       # 3 x [S_local, h, w, 512]
    sums: list              # per level (sum, sum of squares) over ALL S, float64 [h*w, 512]
    pose_embed: torch.Tensor  # [rfn_local, 512]
    shape: tuple            # (rfn_local, an)
    rfn_total: int          # references over all shards


class ViewpointSelector(PackedModule):
    default_cfg = {'selector_angle_num': 5}

    def __init__(self, cfg):
        self.cfg = {**self.default_cfg, **cfg}
        super().__init__()
        self.backbone = VGG11BNParams()
        for name, mod in selector_modules(self.cfg['selector_angle_num']).items():
            setattr(self, name, mod)
        self.refs = None              # SelectorRefs of the object load_ref_imgs / extract_ref_feats loaded
        self.comm = LocalComm()       # gen6d_b200.dist.Comm when the reference axis is sharded over GPUs

    ref_feats_cache = property(lambda self: None if self.refs is None else self.refs.feats_cache)
    ref_sums = property(lambda self: None if self.refs is None else self.refs.sums)
    ref_pose_embed = property(lambda self: None if self.refs is None else self.refs.pose_embed)
    ref_shape = property(lambda self: None if self.refs is None else self.refs.shape)
    rfn_total = property(lambda self: None if self.refs is None else self.refs.rfn_total)

    # ------------------------------------------------------------------ weights
    def _pack(self):
        an = self.cfg['selector_angle_num']
        p = {'vgg': pack_vgg(self.backbone)}
        p['towers'] = []
        for lvl in range(3):
            tower = self.corr_conv_list[lvl]
            p['towers'].append([(ops.pack_conv(tower[s].weight, tower[s].bias, pad=(0, 1, 1)), SEL_TOWER_POST[lvl][s])
                                for s in sorted(SEL_TOWERS[lvl])])
        cf = self.corr_feats_conv
        p['cf0'] = ops.pack_conv(cf[0].weight, cf[0].bias, pad=0)
        p['cf3'] = ops.pack_conv(cf[3].weight, cf[3].bias, pad=0)
        sp = self.score_process
        p['sp0'] = ops.pack_conv(sp[0].weight, sp[0].bias, pad=0, cin_pad=FEAT_PAD)
        p['sp2'] = ops.pack_conv(sp[2].weight, sp[2].bias, pad=0)
        # attention.py:50-68 splits channels as c = d*8 + head; the tiled attention kernel wants each head's 64
        # dims contiguous (c' = head*64 + d).  Permuting the OUTPUT rows of conv_query / conv_key / conv_feats
        # and the INPUT columns of conv_merge once here makes the projections emit / consume that order.
        heads, dh = 8, 64
        hm = torch.arange(512, device=self.device)
        hm = (hm % dh) * heads + hm // dh                     # position c' = h*64 + d  <-  reference channel d*8 + h
        p['atts'] = []
        for att in self.atts:
            pk = {k: linear_as_conv(getattr(att, k).weight[hm], getattr(att, k).bias[hm]) for k in ('conv_query', 'conv_key', 'conv_feats')}
            pk['conv_merge'] = linear_as_conv(att.conv_merge.weight[:, hm], att.conv_merge.bias)
            p['atts'].append(pk | {'ln_w': att.norm.norm.weight.float().contiguous(),
                                   'ln_b': att.norm.norm.bias.float().contiguous()})
        p['mlps'] = [(linear_as_conv(m[0].weight, m[0].bias), linear_as_conv(m[3].weight, m[3].bias)) for m in self.mlps]
        p['score_predict'] = [linear_as_conv(self.score_predict[i].weight, self.score_predict[i].bias) for i in (0, 2)]
        # angle_predict consumes feats.permute(0,1,3,2).reshape(qn, f*an, rfn): channel = f*an + a
        # (selector.py:212-214).  Our per-reference row is [an, FEAT_PAD] flattened (a*FEAT_PAD + f),
        # so permute (and zero-pad) the first layer's input columns once here.
        w0 = self.angle_predict[0].weight.reshape(512, 515, an)            # [o, f, a]
        w0p = torch.zeros(512, an, FEAT_PAD, device=w0.device, dtype=torch.float32)
        w0p[:, :, :515] = w0.permute(0, 2, 1)
        p['angle_predict'] = [linear_as_conv(w0p.reshape(512, an * FEAT_PAD, 1), self.angle_predict[0].bias)] + \
                             [linear_as_conv(self.angle_predict[i].weight, self.angle_predict[i].bias) for i in (2, 4)]
        p['vpe'] = [linear_as_conv(self.view_point_encoder[i].weight, self.view_point_encoder[i].bias) for i in (0, 2, 4)]
        return p

    # ------------------------------------------------------------------ features
    def _feats(self, imgs_norm4):
        """selector.py:113-119: VGG + per-pixel L2 normalisation; input already ImageNet-normalised."""
        return [ops.l2norm_channels(f) for f in vgg_v1(self.packed()['vgg'], imgs_norm4)]

    @staticmethod
    def viewpoints(ref_poses, object_center, object_vert):
        """Normalised viewpoint directions (selector.py:131-147), fp32 on the host: camera centres
        relative to the object in the (x, y, vert) frame anchored on the FIRST reference."""
        ref_poses = torch.as_tensor(ref_poses, dtype=torch.float32).cpu()
        center = torch.as_tensor(object_center, dtype=torch.float32).cpu()
        vert = torch.as_tensor(object_vert, dtype=torch.float32).cpu()
        cam = (-ref_poses[:, :3, :3].permute(0, 2, 1) @ ref_poses[:, :3, 3:])[..., 0] - center[None]
        fwd = cam[0]
        y = torch.linalg.cross(vert, fwd)
        x = torch.linalg.cross(y, vert)
        nrm = lambda v: v / torch.clamp(torch.linalg.norm(v), min=1e-12)
        R = torch.stack([nrm(x), nrm(y), nrm(vert)], 0)
        cam = cam @ R.T
        return cam / torch.clamp(torch.linalg.norm(cam, dim=1, keepdim=True), min=1e-12)

    def _load_nhwc(self, ref_norm4, rfn, an, ref_poses, object_center, object_vert, chunk=64):
        self.refs = self._make_refs(ref_norm4, rfn, an, ref_poses, object_center, object_vert, chunk)
        self.bump_generation()          # captured graphs / worker clones hold pointers to the previous reference set

    def _make_refs(self, ref_norm4, rfn, an, ref_poses, object_center, object_vert, chunk=64):
        """ref_norm4: this rank's references [r0, r1) of the rfn in total, [S_local = (r1-r0)*an (r-major), h, w, 4]
        ImageNet-normalised (selector.py:121-148); ref_poses are those of ALL rfn references.  The callers
        slice the image set BEFORE it is uploaded / converted, so a rank never holds more than its shard.
        -> SelectorRefs (not stored)."""
        p = self.packed()
        rfn_total = rfn
        r0, r1 = self.comm.shard_range(rfn)
        assert ref_norm4.shape[0] == (r1 - r0) * an
        vp_all = self.viewpoints(ref_poses, object_center, object_vert)   # frame anchored on GLOBAL ref 0
        rfn = r1 - r0
        S = rfn * an
        levels = [[], [], []]
        for s0 in range(0, S, chunk):
            for l, f in enumerate(self._feats(ref_norm4[s0:s0 + chunk])):
                levels[l].append(f)
        feats_cache = [torch.cat(lv, 0) if len(lv) > 1 else lv[0] for lv in levels]
        sums = [ops.sel_ref_sums(f.reshape(S, -1, f.shape[-1])) for f in feats_cache]
        # closed-form first-InstanceNorm statistics need the sums over ALL references: one all-reduce at load
        sums = [(self.comm.all_reduce_sum(a), self.comm.all_reduce_sum(b)) for a, b in sums]
        vp = torch.zeros(rfn, 4, dtype=torch.float32)
        vp[:, :3] = vp_all[r0:r1]
        x = vp.to(self.device).reshape(rfn, 1, 1, 4)
        for i, pc in enumerate(p['vpe']):
            x = ops.conv(x, pc, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE)
        return SelectorRefs(feats_cache, sums, x.reshape(rfn, 512), (rfn, an), rfn_total)

    @staticmethod
    def s2_counters_for(refs, device):
        """Fresh completion counters of the fused S2 kernel for one reference record (zero; the kernel leaves them
        zero).  Every record selected against concurrently needs its own."""
        return torch.zeros(3 * refs.shape[0] * refs.shape[1], device=device, dtype=torch.int32)

    def comm_stats(self):
        """Collectives issued by the sharded path (counted on the last eager / capture pass)."""
        return dict(getattr(self.comm, 'calls', {}))

    def _s2_counters(self):
        """Completion counters of the fused S2 kernel: zero between calls (the kernel restores that), private
        to this handle (worker clones run concurrently on other streams and get their own)."""
        n = 3 * self.ref_shape[0] * self.ref_shape[1]
        c = self.__dict__.get('_s2_done')
        if c is None or c.numel() != n or c.device != self.device:
            c = torch.zeros(n, device=self.device, dtype=torch.int32)
            self.__dict__['_s2_done'] = c
        return c

    def _finalize(self, ws, rows_total):
        """InstanceNorm scale / shift from the (sum, sum-of-squares) moments a convolution's epilogue
        produced (fp64).  The group may span GPUs: the moments are all-reduced first, so the statistics are
        exact, not per-shard."""
        return ops.instnorm_finalize(self.comm.all_reduce_sum(ws), rows_total, IN_EPS)

    def _tower_conv(self, level, i, st, Q, S, cat_buf):
        """Convolution i of corr_conv_list[level] (selector.py:27-69) for the Q queries of a batched selection.  st holds
        the tower's input x, prologue and its operands.  Every layer has a prologue; prenorm applies it in a split pass
        over the input, so the A operand arrives by TMA instead of a per-tap gather.  The 16x16 level-0 layers, which
        the A-reuse kernel would take, run on the persistent kernel in that kernel's K order (reuse_im2col), so the
        result is the same bit for bit.
        The first layer forms q (.) ref from the one reference stack: one call per query, each writing its query's rows
        of the batched output and its group of the moments.  Every later layer is one call over the Q*S images, the
        queries' InstanceNorm groups of S images each, with the K splits planned for one query's rows (plan_rows), so
        every query's output is the bits a call of that query alone gives.  -> (y, moments [Q, Cout, 2], rows per
        query), or None for the last layer (written into cat_buf)."""
        pc, post = self.packed()['towers'][level][i]
        x = st['x']
        kw = dict(prenorm=True, reuse_im2col=True, fold_splits=True)
        if i == 0:
            rows = x.shape[0] * x.shape[1] * x.shape[2]                # stride-1 same-size convolution, one query
            y = torch.empty(Q * x.shape[0], x.shape[1], x.shape[2], pc.cout, device=x.device, dtype=torch.float32)
            ws = [ops.conv(x, pc, prologue=ops.PRO_CORR, pro_scale=st['ps'][q], pro_shift=st['pb'][q], group_rows=S,
                           out=y[q * S:(q + 1) * S], stats_rows=rows, **kw)[1] for q in range(Q)]
            return y, (ws[0] if Q == 1 else torch.cat(ws, 0)), rows
        rows = x.shape[0] * x.shape[1] * x.shape[2] // Q
        if i + 1 == len(self.packed()['towers'][level]):
            ops.conv(x, pc, prologue=st['pro'], pro_scale=st['ps'], pro_shift=st['pb'], group_rows=S, out=cat_buf,
                     out_coff=256 * level, plan_rows=rows, **kw)
            return None
        return ops.conv(x, pc, prologue=st['pro'], pro_scale=st['ps'], pro_shift=st['pb'], group_rows=S, stats_rows=rows,
                        plan_rows=rows, **kw) + (rows,)

    @staticmethod
    def _tower_next(st, post, y, ps, pb):
        """The normalisation (and ReLU) of InstanceNorm3d is applied by the next conv's loader.  MaxPool commutes with
        the positive-slope affine, so pooling the raw tensor first is exact."""
        st['ps'], st['pb'] = ps, pb
        st['pro'] = ops.PRO_AFFINE_RELU if 'r' in post else ops.PRO_AFFINE
        st['x'] = ops.maxpool2x2(y) if 'p' in post else y

    def _tower_state(self, q, ref, s1, s2, S_total):
        """A tower's input: the reference stack and each query's q (.) ref prologue (first InstanceNorm3d folded in)."""
        Q, h, w, c = q.shape
        pro = [ops.sel_corr_prologue(q[i].reshape(h * w, c), s1, s2, S_total, IN_EPS) for i in range(Q)]
        return {'x': ref, 'ps': [a for a, _ in pro], 'pb': [b for _, b in pro]}

    def _tower(self, level, st, Q, cat_buf, S, refs):
        """corr_conv_list[level] on the implicit correlation volume of Q queries, one layer after the other."""
        convs = self.packed()['towers'][level]
        for i, (_, post) in enumerate(convs):
            res = self._tower_conv(level, i, st, Q, S, cat_buf)
            if res is None:
                break
            y, ws, rows = res
            # InstanceNorm3d statistics over (S, h, w) of the raw conv output, per query
            ps, pb = self._finalize(ws, rows // refs.shape[0] * refs.rfn_total)
            self._tower_next(st, post, y, ps, pb)

    def _towers_sharded(self, q_feats, cat_buf, Q, S, S_total, refs):
        """The three towers with the reference axis sharded over GPUs, ROUND-synchronous: round r runs the
        r-th convolution of every tower that still has one (concurrently, on branch streams), then ONE
        all-reduce carries the InstanceNorm moments of all of them and of all Q queries (5 rounds for the 6 + 4 + 2
        convolutions instead of 9 per-layer all-reduces; SURVEY 8e).  Same arithmetic as _tower."""
        towers = self.packed()['towers']
        nbr = 3 if self.comm.capturable else 1
        state = [self._tower_state(q, ref, s1, s2, S_total)
                 for q, ref, (s1, s2) in zip(q_feats, refs.feats_cache, refs.sums)]
        keep = []
        for i in range(max(len(t) for t in towers)):
            br = Branches(nbr)          # forks from the main stream: after the previous round's finalize / pool kernels
            pend = []
            for l, st in enumerate(state):
                if i >= len(towers[l]):
                    continue
                res = br.run(l, lambda l=l, st=st: self._tower_conv(l, i, st, Q, S, cat_buf))
                if res is not None:
                    pend.append((st, towers[l][i][1], res))
            br.join()
            if not pend:
                continue
            flat = torch.cat([ws.reshape(-1) for _, _, (_, ws, _) in pend]) if len(pend) > 1 else pend[0][2][1].reshape(-1)
            flat = self.comm.all_reduce_sum(flat)                 # one collective for every tower's moments of this round
            o = 0
            for st, post, (y, ws, rows) in pend:
                n = ws.numel()
                ps, pb = ops.instnorm_finalize(flat[o:o + n].reshape(ws.shape), rows // refs.shape[0] * refs.rfn_total, IN_EPS)
                o += n
                keep.append((y, ws))
                self._tower_next(st, post, y, ps, pb)

    def _select_batch(self, q_feats, refs=None, counters=None):
        """selector.py:177-215 for Q queries against one reference record.  q_feats: 3 x [Q, h, w, 512].
        -> logits [Q, rfn], angles [Q, rfn], S2 scores [Q, 3, S].  Queries run in chunks of SEL_QUERY_CHUNK: the layers
        after each tower's first run once per chunk over all its queries, each query's rows bit for bit what a chunk of
        that query alone gives.  refs: the SelectorRefs to select against (default: the module's own); with any other
        record, `counters` are that record's own S2 counters (s2_counters_for), never the module's or another record's."""
        if refs is None:
            refs, counters = self.refs, self._s2_counters()
        rfn, an = refs.shape
        if counters is None or counters.numel() != 3 * rfn * an:
            raise ValueError('_select_batch: a reference record other than the module\'s needs its own S2 counters [3*S]')
        Q = q_feats[0].shape[0]
        if Q <= SEL_QUERY_CHUNK:
            return self._select_chunk(q_feats, refs, counters)
        parts = [self._select_chunk([f[q0:q0 + SEL_QUERY_CHUNK] for f in q_feats], refs, counters)
                 for q0 in range(0, Q, SEL_QUERY_CHUNK)]
        return tuple(torch.cat(t, 0) for t in zip(*parts))

    def _select_chunk(self, q_feats, refs, counters):
        p = self.packed()
        Q = q_feats[0].shape[0]
        rfn, an = refs.shape
        S = rfn * an
        S_total = refs.rfn_total * an
        dev = self.device
        cat_buf = torch.empty(Q * S, 4, 4, 768, device=dev, dtype=torch.float32)
        feats = torch.empty(Q * S, FEAT_PAD, device=dev, dtype=torch.float32)  # cols 0-511: cf3, 512-514 + pad: vp_norm
        scores = torch.empty(Q, 3, S, device=dev, dtype=torch.float32)
        ref_rows = [r.reshape(S, -1, r.shape[-1]) for r in refs.feats_cache]
        for q in range(Q):
            ops.sel_corr_score3(ref_rows, [f[q].reshape(-1, f.shape[-1]) for f in q_feats], counters=counters, out=scores[q])
        if self.comm.world == 1:
            br = Branches(3)                                # the three towers only meet in cat_buf
            keep = []

            def one_level(l, q, ref, s1, s2):
                st = self._tower_state(q, ref, s1, s2, S_total)
                keep.append(st)
                self._tower(l, st, Q, cat_buf, S, refs)

            for l, (q, ref, (s1, s2)) in enumerate(zip(q_feats, refs.feats_cache, refs.sums)):
                br.run(l, lambda l=l, q=q, ref=ref, s1=s1, s2=s2: one_level(l, q, ref, s1, s2))
            br.join()
        else:
            self._towers_sharded(q_feats, cat_buf, Q, S, S_total, refs)
        # corr_feats_conv (selector.py:71-77): 1x1 768->512, IN, ReLU, 1x1 512->512, AvgPool(4,4).
        # The second 1x1 conv is linear, so the 4x4 average is taken first (16x less work).
        y, ws = ops.conv(cat_buf, p['cf0'], stats_rows=S * 16, plan_rows=S * 16)
        ps, pb = self._finalize(ws, S_total * 16)
        y = ops.avgpool_affine(y.reshape(Q * S * 16, 512), 16, ps, pb, rows_per_group=S * 16, act=ops.ACT_RELU)
        ops.conv(y.reshape(Q * S, 1, 1, 512), p['cf3'], out=feats.reshape(Q * S, 1, 1, FEAT_PAD), out_coff=0, plan_rows=S)
        if self.comm.world == 1:
            for q in range(Q):
                ops.sel_vp_norm(scores[q], feats[q * S:(q + 1) * S], 512, IN_EPS)         # vp_norm, selector.py:201
        else:   # InstanceNorm2d over ALL (rfn, an): gather the 3*S_total scores, normalise, keep our rows
            all_scores = self.comm.all_gather_cat(scores, dim=2).contiguous()
            tmp = torch.empty(Q, S_total, 4, device=dev, dtype=torch.float32)
            for q in range(Q):
                ops.sel_vp_norm(all_scores[q], tmp[q], 0, IN_EPS)
            r0, _ = self.comm.shard_range(refs.rfn_total)
            feats.reshape(Q, S, FEAT_PAD)[:, :, 512:516] = tmp[:, r0 * an:r0 * an + S]
        x = ops.conv(feats.reshape(Q * S, 1, 1, FEAT_PAD), p['sp0'], act=ops.ACT_RELU, plan_rows=S)
        x = ops.conv(x, p['sp2'], plan_rows=S).reshape(Q * rfn, an, 512)
        sf = torch.empty(Q * rfn, 512, device=dev, dtype=torch.float32)
        for q in range(Q):                                              # selector.py:203-204
            ops.sel_max_angle_add(x[q * rfn:(q + 1) * rfn], refs.pose_embed, out=sf[q * rfn:(q + 1) * rfn])
        # everything below couples all references (attention, InstanceNorm1d over rfn): gather the
        # per-reference score features once ([rfn,512] = 128 KB per query at 64 refs) and run the tail replicated
        sf = self.comm.all_gather_cat(sf.reshape(Q, rfn, 512), dim=1).contiguous()
        rfn_local, rfn = rfn, refs.rfn_total
        sf = sf.reshape(Q * rfn, 512)
        for att, (m0, m3) in zip(p['atts'], p['mlps']):
            x4 = sf.reshape(Q * rfn, 1, 1, 512)
            qv = ops.conv(x4, att['conv_query'], plan_rows=rfn).reshape(Q * rfn, 512)
            kv = ops.conv(x4, att['conv_key'], plan_rows=rfn).reshape(Q * rfn, 512)
            vv = ops.conv(x4, att['conv_feats'], plan_rows=rfn).reshape(Q * rfn, 512)
            msg = torch.empty_like(qv)
            for q in range(Q):
                r = slice(q * rfn, (q + 1) * rfn)
                ops.attention(qv[r], kv[r], vv[r], heads=8, head_major=True, out=msg[r])
            msg = ops.conv(msg.reshape(Q * rfn, 1, 1, 512), att['conv_merge'], plan_rows=rfn).reshape(Q * rfn, 512)
            msg = ops.layernorm(msg, att['ln_w'], att['ln_b'], 1e-5)
            y = ops.conv(torch.cat([sf, msg], 1).reshape(Q * rfn, 1, 1, 1024), m0, plan_rows=rfn)
            ps, pb = ops.instnorm_stats(y, rows_per_group=rfn, eps=IN_EPS)      # InstanceNorm1d over rfn, per query
            y = ops.conv(y, m3, prologue=ops.PRO_AFFINE_RELU, pro_scale=ps, pro_shift=pb, group_rows=rfn, plan_rows=rfn)
            ps, pb = ops.instnorm_stats(y, rows_per_group=rfn, eps=IN_EPS)
            y = ops.affine_act(y.reshape(Q * rfn, 512), ps, pb, rows_per_group=rfn, act=ops.ACT_RELU)
            sf = ops.add(y, sf)
        x = ops.conv(sf.reshape(Q * rfn, 1, 1, 512), p['score_predict'][0], act=ops.ACT_RELU, plan_rows=rfn)
        logits = ops.conv(x, p['score_predict'][1], plan_rows=rfn).reshape(Q, rfn)
        x = feats.reshape(Q * rfn_local, 1, 1, an * FEAT_PAD)           # angles are per-reference: local
        for i, pc in enumerate(p['angle_predict']):
            x = ops.conv(x, pc, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE, plan_rows=rfn_local)
        angles = self.comm.all_gather_cat(x.reshape(Q, rfn_local), dim=1)
        return logits, angles, scores

    def _select_nhwc(self, que_norm4):
        if self.ref_feats_cache is None:
            raise RuntimeError('ViewpointSelector: load_ref_imgs / extract_ref_feats must be called first')
        return self._select_batch(self._feats(que_norm4))

    def _select_u8(self, u8):
        """uint8 crop(s) on the device -> (ref_idx [qn], (angle, logit) [qn,2], logits [qn,rfn])."""
        logits, angles, _ = self._select_nhwc(ops.preprocess_u8(u8, out_c=4, imagenet_norm=True))
        idx, out = ops.sel_parse(logits, angles)
        return idx, out, logits

    # ------------------------------------------------------------------ reference tensor API
    def extract_ref_feats(self, ref_imgs, ref_poses, object_center, object_vert, is_train=False):
        """ref_imgs [an,rfn,3,h,w] in [0,1] (selector.py:121-148; is_train=False path only)."""
        if is_train:
            raise NotImplementedError('inference-only build: random forward-view selection is a training feature')
        with torch.no_grad():
            an, rfn, _, h, w = ref_imgs.shape
            r0, r1 = self.comm.shard_range(rfn)
            x = ref_imgs[:, r0:r1].permute(1, 0, 2, 3, 4).reshape((r1 - r0) * an, 3, h, w).float().contiguous()
            x = ops.imagenet_norm(ops.nchw_to_nhwc(x), out_c=4)
            self._load_nhwc(x, rfn, an, ref_poses, object_center, object_vert)

    def compute_view_point_feats(self, que_imgs):
        """que_imgs [qn,3,h,w] in [0,1] -> logits [qn,rfn], angles [qn,rfn] (selector.py:177-215)."""
        with torch.no_grad():
            x = ops.imagenet_norm(ops.nchw_to_nhwc(que_imgs.float().contiguous()), out_c=4)
            logits, angles, _ = self._select_nhwc(x)
        return logits, angles

    def forward(self, data):
        self.extract_ref_feats(data['ref_imgs'], data['ref_imgs_info']['poses'], data['object_center'],
                               data['object_vert'], 'eval' not in data)
        logits, angles = self.compute_view_point_feats(data['que_imgs_info']['imgs'])
        return {'ref_vp_logits': logits, 'angles_pr': angles}

    # ------------------------------------------------------------------ reference numpy API
    def load_ref_imgs(self, ref_imgs, ref_poses, object_center, object_vert):
        """@param ref_imgs: uint8 [an,rfn,h,w,3]; ref_poses [rfn,3,4]; object_center [3]; object_vert [3]
        (selector.py:150-163)"""
        self.refs = self.make_refs(ref_imgs, ref_poses, object_center, object_vert)
        self.bump_generation()          # captured graphs / worker clones hold pointers to the previous reference set

    def make_refs(self, ref_imgs, ref_poses, object_center, object_vert):
        """What load_ref_imgs computes, returned as a SelectorRefs instead of stored."""
        with torch.no_grad():
            an, rfn, h, w, _ = ref_imgs.shape
            r0, r1 = self.comm.shard_range(rfn)
            u8 = torch.from_numpy(np.ascontiguousarray(ref_imgs[:, r0:r1].transpose(1, 0, 2, 3, 4))).to(self.device)
            u8 = u8.reshape((r1 - r0) * an, h, w, 3)            # one-off load: no pinned staging ring for ~100s of MB
            x = ops.preprocess_u8(u8, out_c=4, imagenet_norm=True)
            return self._make_refs(x, rfn, an, ref_poses.astype(np.float32), object_center.astype(np.float32),
                                   object_vert.astype(np.float32))

    def _select_warped(self, size):
        def fn(jobs):
            crop = ops.warp_affine_u8(jobs, jobs.numel() // ops.WARP_JOB_BYTES, size, size)
            return (crop,) + tuple(self._select_u8(crop))
        return fn

    def select_from_frame(self, frame_dev, M, size):
        """estimator.py:184-186 in one device stage: cut the detection crop out of the frame with the
        2x3 similarity M (g6d_warp_affine_u8, bit-exact with the reference's cv2.warpAffine), then
        select_que_imgs on it.  frame_dev: uint8 [h,w,3] on the device.  Returns the select_que_imgs
        dict plus 'que_imgs' (the crop, uint8 [1,size,size,3], as the reference hands it on)."""
        from .. import geometry as G
        fn = self._select_warped(size)
        with torch.no_grad():
            jobs = self._to_dev(G.pack_warp_jobs([frame_dev], [G.affine_dst_to_src(M)]))
            if self.comm.capturable:
                crop, idx, out, logits = self.stages.run(f'select_warp{size}', fn, [jobs])
            else:
                crop, idx, out, logits = fn(jobs)           # host-staged collectives inside: run eagerly
            crop, idx, out, logits = [self._to_host(t) for t in (crop, idx, out, logits)]
        return {'ref_idx': idx, 'angles': out[:, 0].copy(), 'scores': logits, 'que_imgs': crop}

    def select_from_frames(self, frames_dev, Ms, size):
        """Batched select_from_frame: crop i is cut out of frames_dev[i] (uint8 [qn,h,w,3] on the device)
        with the 2x3 similarity Ms[i]; one stage (one graph launch, one D2H) for the whole batch."""
        from .. import geometry as G
        fn = self._select_warped(size)
        with torch.no_grad():
            jobs = self._to_dev(G.pack_warp_jobs([frames_dev[i] for i in range(len(Ms))], [G.affine_dst_to_src(M) for M in Ms]))
            if self.comm.capturable:
                crop, idx, out, logits = self.stages.run(f'select_warp{size}', fn, [jobs])
            else:
                crop, idx, out, logits = fn(jobs)
            crop, idx, out, logits = [self._to_host(t) for t in (crop, idx, out, logits)]
        return {'ref_idx': idx, 'angles': out[:, 0].copy(), 'scores': logits, 'que_imgs': crop}

    def select_que_imgs(self, que_imgs):
        """@param que_imgs: uint8 [qn,h,w,3] -> {'ref_idx': i64 [qn], 'angles': f32 [qn], 'scores': f32 [qn,rfn]}
        (selector.py:165-175; the angle is returned un-rescaled, as the reference does)"""
        with torch.no_grad():
            u8 = self._to_dev(que_imgs)
            if self.comm.capturable:    # NCCL collectives are captured with the kernels; gloo (host-staged) runs eagerly
                idx, out, logits = self.stages.run('select', self._select_u8, [u8])
            else:
                idx, out, logits = self._select_u8(u8)
            idx, out, logits = self._to_host(idx), self._to_host(out), self._to_host(logits)
        return {'ref_idx': idx, 'angles': out[:, 0].copy(), 'scores': logits}
