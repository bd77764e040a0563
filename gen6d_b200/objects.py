"""Several objects per frame over one set of networks.

Gen6D is model-free: one checkpoint serves every object, and an object is only its reference state (the detector's
correlation kernels, the selector's reference stack, the refiner's database images).  An ObjectSet
(Gen6DEstimator.object_set()) keeps that state per object, next to the estimator's own, and poses every object on the
same frames as ONE captured graph with one synchronising read:

  upload -> ONE detection stage for all objects (the query's VGG pyramid once per scale, one correlation GEMM per level
  over the objects' concatenated kernels, g6d_det_corr_rowsum_objects, then score fusion / heads / argmax on K*qn
  "queries") -> the K*qn selector crops in one warp and one crop VGG, each object's selection against its own reference
  stack -> refine_iter x (the objects' refinement problems in one launch, ONE refiner stage over all K*qn poses, the
  objects' updates in one launch; g6d_glue_*_objects).

Rows are object-major (object, frame) everywhere after the correlation, so each object's detections, crops and poses are
a contiguous slice whose row i is frame i, which is the layout the g6d_glue_* kernels take.  ObjectSet.tracker() follows
the set's objects through videos (gen6d_b200/track.py ObjectTracker), ObjectSet.instance_tracker() every instance of
each (gen6d_b200/instance_track.py ObjectInstanceTracker).
"""
from functools import partial

import numpy as np
import torch

from . import boxes as B
from . import frames as F
from . import glue
from . import instances
from . import ops
from . import verify
from .graphs import StageCache


def require_device_pipeline(est, what):
    """The estimator features an object set and predict_instances need: a refiner, an unsharded selector, device warps."""
    if est.refiner is None:
        raise ValueError(f'{what} refines every pose: the estimator needs a refiner')
    if getattr(est.selector.comm, 'world', 1) > 1:
        raise ValueError(f'{what} does not shard the selector: the estimator\'s selector is sharded over GPUs')
    if est.cfg['host_warps']:
        raise ValueError(f"{what} cuts its crops on the device: cfg['host_warps'] must be False")


class _Object:
    """One object's reference state: a record per network module plus its glue tables on the device."""

    def __init__(self, det, sel, ref, ref_info, tables, counters, weights_gen):
        self.det, self.sel, self.ref = det, sel, ref
        self.ref_info, self.tables, self.counters = ref_info, tables, counters
        self.weights_gen = weights_gen


class ObjectSet:
    """Objects sharing one estimator's networks; see Gen6DEstimator.object_set().

    Per object the device holds about the selector's reference stack (220 MB at 64 views x 5 angles), the detector's
    kernels (tens of MB) and the object's database images (66 MB for a 72-view 480x640 object)."""

    def __init__(self, est):
        require_device_pipeline(est, 'an object set')
        self.est = est
        self._objects = {}
        self._kernels = None            # the objects' detector kernels concatenated (rebuilt when membership changes)
        self.membership = 0             # counts add / remove: a tracker made before a change is stale
        self.stages = StageCache()      # the set's prediction graph

    # -------------------------------------------------------------- membership
    @property
    def names(self):
        return list(self._objects)

    def __len__(self):
        return len(self._objects)

    def __contains__(self, name):
        return name in self._objects

    def add(self, name, database):
        """Compute `database`'s reference state (what est.build(database, 'all') computes) and store it under `name`.
        A reference-repo database is wrapped as build() does; cfg['device_build'] is honoured."""
        from .database import as_object_database
        if name in self._objects:
            raise ValueError(f'object {name!r} is already in the set')
        est = self.est
        database = as_object_database(database)
        v = est._reference_views(database)
        det_imgs = v['imgs'][:est.cfg['det_ref_view_num']]
        if self._objects:
            rfn = next(iter(self._objects.values())).det.rfn
            if len(det_imgs) != rfn:
                raise ValueError(f'object {name!r} has {len(det_imgs)} detector reference views, the set\'s objects have {rfn}: '
                                 'the detection correlation concatenates the objects\' kernels, so every object needs '
                                 f"det_ref_view_num ({est.cfg['det_ref_view_num']}) views; a database with fewer views "
                                 'than that gives fewer')
        weights_gen = est._weights_generation()
        det = est.detector.make_refs_u8(det_imgs)
        sel = est.selector.make_refs(v['ref_imgs'], v['poses'], v['center'], v['vert'])
        ref = est.refiner.make_refs(database, v['ids_all'])
        ref_info = {k: v[k] for k in ('imgs', 'ref_imgs', 'Ks', 'poses', 'center', 'ref_ids')}
        tables = est._device_tables(ref_info, ref)          # synchronises: the state is complete before any use
        counters = est.selector.s2_counters_for(sel, est.selector.device)
        self._objects[name] = _Object(det, sel, ref, ref_info, tables, counters, weights_gen)
        self._membership_changed()

    def remove(self, name):
        if name not in self._objects:
            raise ValueError(f'object {name!r} is not in the set (objects: {self.names})')
        del self._objects[name]
        self._membership_changed()

    def _membership_changed(self):
        self.membership += 1
        self._kernels = None
        self.stages.clear()             # the graph captured the previous objects' state

    def _check(self):
        if not self._objects:
            raise ValueError('the object set is empty: add objects first')
        gen = self.est._weights_generation()
        stale = [n for n, o in self._objects.items() if o.weights_gen != gen]
        if stale:
            raise RuntimeError(f'objects {stale} are stale: the networks\' weights changed since they were added, and their '
                               'reference features were computed with the old weights; remove and add them again')

    def _detector_kernels(self):
        if self._kernels is None:
            with torch.no_grad():
                self._kernels = self.est.detector.pack_kernels([o.det.center_feats for o in self._objects.values()])
        return self._kernels

    # -------------------------------------------------------------- prediction
    def _detect(self, u8, return_taps=False):
        """uint8 frames [qn,h,w,3] -> detector outputs of K*qn object-major rows (and taps)."""
        objs = list(self._objects.values())
        det = self.est.detector
        o = det._detect_objects_nhwc(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False), self._detector_kernels(),
                                     len(objs), objs[0].det.rfn, return_taps)
        out, _ = ops.det_parse(o['score_predict'], o['scale_predict'], o['offset_predict'], det.pool_ratio)
        return out, o

    def _initial_poses_device_fn(self, detect=None):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> the shared detection, each slot's selection and the initial poses:
        (poses f64 [S*qn,12] slot-major, det [S*qn,4], [(sel_idx, sel_out, logits)] per slot, crops u8 [S*qn,res,res,3]).
        detect(frames) -> det [S*qn,4] is the detection step, slot s being object s % K: the argmax of each object's map
        (S = K) by default, _peaks_detect_fn's instances (S = M*K) for predict_instances."""
        est = self.est
        objs = list(self._objects.values())
        K, res = len(objs), est.cfg['ref_resolution']
        sel = est.selector

        def fn(frames, cams):
            qn = frames.shape[0]
            rows = lambda t, o: t[o * qn:(o + 1) * qn]
            cat = lambda ts: ts[0] if len(ts) == 1 else torch.cat(ts, 0)
            det = F.per_size(lambda u8: self._detect(u8)[0], frames) if detect is None else detect(frames)   # [S*qn,4]: x, y, scale, score
            S = det.shape[0] // qn
            jobs = cat([ops.glue_detection_jobs(rows(det, s), frames, res) for s in range(S)])
            crop = ops.warp_affine_u8(jobs, S * qn, res, res)
            feats = sel._feats(ops.preprocess_u8(crop, out_c=4, imagenet_norm=True))  # the crop VGG once for all slots
            poses, sels = [], []
            for s in range(S):
                ob = objs[s % K]
                logits, angles, _ = sel._select_batch([rows(f, s) for f in feats], ob.sel, ob.counters)
                idx, sel_out = ops.sel_parse(logits, angles)
                sels.append((idx, sel_out, logits))
                poses.append(ops.glue_initial_poses(rows(det, s), idx, sel_out, ob.tables['refs'], cams))
            return cat(poses), det, sels, crop                                       # poses [S*qn,12], slot-major
        return fn

    def _peaks_detect_fn(self, M, radius, nms_iou, min_score):
        """The detection step of predict_instances: the shared pyramid and correlation of _detect, then g6d_det_parse_peaks
        on the K*qn maps -> det [M*K*qn,4] (slot m*K + o is instance m of object o).  `extra` receives valid int32 [M*K*qn]
        and count int32 [K*qn] when the returned function runs."""
        est = self.est
        det_mod, box = est.detector, float(est.cfg['ref_resolution'])
        objs = list(self._objects.values())
        extra = []

        def one_size(u8):
            o = det_mod._detect_objects_nhwc(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False), self._detector_kernels(),
                                             len(objs), objs[0].det.rfn)
            det, _, valid, count = ops.det_parse_peaks(o['score_predict'], o['scale_predict'], o['offset_predict'], M, radius,
                                                       nms_iou, box, min_score, det_mod.pool_ratio)
            return det.reshape(-1, 4), valid.reshape(-1), count

        def detect(frames):
            det, valid, count = F.per_size(one_size, frames)                       # once per frame size (row f13)
            extra[:] = [valid, count]
            return det
        return detect, extra

    def _predict_device_fn(self, detect=None, instances=1):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> every stage, back to back, as device tensors: (chain f64
        [refine_iter+1, S*qn, 12] of slot-major poses, det [S*qn,4], [(sel_idx, sel_out, logits)] per slot, crops u8
        [S*qn, res, res, 3]) with S = instances*K slots, slot s being object s % K (detect: see _initial_poses_device_fn)."""
        est = self.est
        objs = list(self._objects.values())
        iters, R = est.cfg['refine_iter'], objs[0].tables['tables']['ref_num']
        views = [ob.tables['views'] for ob in objs] * instances
        initial, refine = self._initial_poses_device_fn(detect), est.refiner._refine_warped(128)

        def fn(frames, cams):
            poses, det, sels, crop = initial(frames, cams)
            chain = [poses]
            for it in range(iters):
                jobs_r, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_objects(views, R, cams, frames, poses,
                                                                                                       it > 0)
                out = refine(jobs_r, que_K, que_pose, ref_Ks, ref_poses)              # one refiner stage for all S*qn poses
                poses = ops.glue_apply_refinements_objects(views, que_pose, que_K, rect, out)
                chain.append(poses)
            return torch.stack(chain, 0), det, sels, crop
        return fn

    def _predict_fn(self):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> (packed results f64 as bytes ++ crops u8): every stage, back to back."""
        stages, K = self._predict_device_fn(), len(self._objects)

        def fn(frames, cams):
            qn = frames.shape[0]
            chain, det, sels, crop = stages(frames, cams)
            parts = []
            for o in range(K):
                idx, sel_out, logits = sels[o]
                parts += [chain[:, o * qn:(o + 1) * qn], det[o * qn:(o + 1) * qn], idx, sel_out, logits]
            packed = torch.cat([t.reshape(-1).to(torch.float64) for t in parts])
            return torch.cat([packed.view(torch.uint8), crop.reshape(-1)])
        return fn

    def predict(self, que_imgs, que_Ks):
        """Every object's pose on the same qn frames (uint8 [h,w,3], of one size or several: row f13; que_Ks [qn,3,3]).
        Returns {name: (poses [qn,3,4], inter)}: inter has the keys and shapes of predict_batch's device-glue inter, plus
        'det_score' [qn], the maximum of that object's detection score map (is the object in the frame at all).
        que_imgs may be device frames (CUDA RGB tensors, frames.NV12), with predict_batch's rules (row f14)."""
        self._check()
        est = self.est
        qn, res, iters = len(que_imgs), est.cfg['ref_resolution'], est.cfg['refine_iter']
        if qn == 0 or len(que_Ks) != qn:
            raise ValueError(f'predict: {qn} frames and {len(que_Ks)} intrinsics; need one K per frame and at least one frame')
        imgs = F.as_frames(que_imgs, 'predict', est.detector)
        if F.is_mixed(imgs):
            F.check_frames(imgs, que_Ks, 'predict')
        det = est.detector
        with torch.no_grad():
            name, fn, fin = F.stage(det, 'predict', self._predict_fn(), imgs)
            cams = det._to_dev(glue.cameras(np.stack([np.asarray(K) for K in que_Ks], 0)))
            buf = self.stages.run(name, fn, fin + [cams])
            host = det._to_host(buf)                                       # the call's one synchronising read
        crop_bytes = len(self._objects) * qn * res * res * 3
        f64 = host[:len(host) - crop_bytes].view(np.float64)
        crops = host[len(host) - crop_bytes:].reshape(len(self._objects), qn, res, res, 3)
        out, off = {}, 0
        for o, (name, ob) in enumerate(self._objects.items()):
            n_sel = len(ob.ref_info['poses'])

            def take(n):
                nonlocal off
                off += n
                return f64[off - n:off]
            chain = take((iters + 1) * qn * 12).reshape(iters + 1, qn, 3, 4)
            d = take(qn * 4).reshape(qn, 4).astype(np.float32)
            idx = take(qn).astype(np.int64)
            sel_out = take(qn * 2).reshape(qn, 2).astype(np.float32)
            logits = take(qn * n_sel).reshape(qn, n_sel).astype(np.float32)
            refined = [c.astype(np.float32) for c in chain[1:]]
            inter = {'det_position': d[:, :2].copy(), 'det_scale_r2q': d[:, 2].copy(), 'det_score': d[:, 3].copy(),
                     'det_que_img': crops[o].copy(), 'sel_angle_r2q': sel_out[:, 0].copy(), 'sel_scores': logits,
                     'sel_ref_idx': idx, 'refine_poses': [chain[0].copy()] + refined}
            out[name] = (refined[-1] if refined else chain[0].copy(), inter)
        return out

    def _instances_fn(self, M, radius, nms_iou, min_score, boxes=None):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> packed results of predict_instances (the M*K slots' chain, detections,
        per-slot selections, the peak masks and counts, then the crops).  boxes: a boxes.Detect, the detection step from
        caller boxes instead of the maps and peaks."""
        detect, extra = (boxes, boxes.extra) if boxes is not None else self._peaks_detect_fn(M, radius, nms_iou, min_score)
        stages = self._predict_device_fn(detect, M)

        def fn(frames, cams):
            chain, det, sels, crop = stages(frames, cams)
            return instances.pack([chain, det] + [t for sel in sels for t in sel] + extra, crop)
        return fn

    def predict_instances(self, que_imgs, que_Ks, max_instances=4, min_score=None, nms_iou=0.3, peak_radius=1, boxes=None):
        """Every instance of every object on the same qn frames: Gen6DEstimator.predict_instances for each object of the set,
        with the shared query pyramid and correlation of predict().  Slot (m, o) -- instance m of object o -- goes through
        its own crop and object o's selection; a refinement step over the K*M*qn rows is one refiner stage.  Returns
        {name: (poses [qn,M,3,4], inter)} with predict_instances' keys.  Rows of instances that were not found are computed
        and returned, masked by inter['instance_valid'].  One captured graph per argument set and frame shape, one read.
        que_imgs may be device frames, with predict_batch's rules (row f14).
        boxes (row f19): every object's instances from another detector, one dict {object name: boxes} per frame, the
        boxes as Gen6DEstimator.predict_instances takes them; an object missing from a frame's dict has no boxes there
        (instance_count 0), and a name not in the set is a ValueError.  The detector runs no kernel; min_score, nms_iou
        and peak_radius do not apply and are not part of the box graphs' key."""
        self._check()
        key = instances.check_args(max_instances, nms_iou, peak_radius, min_score)
        est = self.est
        M, K = key[0], len(self._objects)
        qn, res, iters = len(que_imgs), est.cfg['ref_resolution'], est.cfg['refine_iter']
        if qn == 0 or len(que_Ks) != qn:
            raise ValueError(f'predict_instances: {qn} frames and {len(que_Ks)} intrinsics; need one K per frame and at least one frame')
        imgs = F.as_frames(que_imgs, 'predict_instances', est.detector)
        if F.is_mixed(imgs):
            F.check_frames(imgs, que_Ks, 'predict_instances')
        det = est.detector
        table = None if boxes is None else B.for_objects(boxes, self.names, qn, 'predict_instances', det.device)
        with torch.no_grad():
            if table is None:
                name, fn, tail = ('instances',) + key, self._instances_fn(*key), []
            else:
                dt = B.Detect(M, K, K * qn, table.N, B.inv_box_size(res))
                name, fn = B.graph_name(('instances', M), table.N), dt.bind(self._instances_fn(*key, boxes=dt))
                tail = [table.upload(det)]
            name, fn, fin = F.stage(det, name, fn, imgs)
            cams = det._to_dev(glue.cameras(np.stack([np.asarray(K_) for K_ in que_Ks], 0)))
            buf = self.stages.run(name, fn, fin + [cams] + tail)
            host = det._to_host(buf)                                       # the call's one synchronising read
        S = M * K
        rd = instances.Unpacker(host, S * qn * res * res * 3)
        chain = rd.take((iters + 1) * S * qn * 12).reshape(iters + 1, M, K, qn, 12)
        dets = rd.take(S * qn * 4).reshape(M, K, qn, 4)
        objs = list(self._objects.values())
        sels = [(rd.take(qn), rd.take(qn * 2), rd.take(qn * len(objs[s % K].ref_info['poses']))) for s in range(S)]
        valid = rd.take(S * qn).reshape(M, K, qn)
        count = rd.take(K * qn).reshape(K, qn)
        crops = rd.crops.reshape(M, K, qn, res, res, 3)
        out = {}
        for o, name in enumerate(self._objects):
            mine = [sels[m * K + o] for m in range(M)]
            cat = lambda i: np.concatenate([s[i] for s in mine])
            out[name] = instances.inter_of(chain[:, :, o].reshape(iters + 1, M * qn, 12), dets[:, o], cat(0), cat(1), cat(2),
                                           valid[:, o], count[o], crops[:, o].reshape(M * qn, res, res, 3), M, qn)
        return out

    def _verify_fn(self, key, M=1):
        """The verification nodes (verify.nodes) of the set's objects, each object's windows detected against its own
        references: the launches of Gen6DEstimator.verify_poses on an estimator built on that object.  M: row groups per
        object (an instance tracker's slots)."""
        objs = list(self._objects.values())
        det = self.est.detector
        return verify.nodes(self.est, [ob.tables['refs'] for ob in objs], [partial(det._detect_u8, refs=ob.det) for ob in objs], key,
                            M)

    def verify_poses(self, que_imgs, que_Ks, poses, lost_score=None, lost_gate=None):
        """Gen6DEstimator.verify_poses for every object of the set on the same qn frames: poses {name: [qn,3,4]} for every
        object (one dtype for all) -> {name: verify_poses' dict}.  One captured graph, one read."""
        self._check()
        key = verify.check_thresholds(lost_score, lost_gate)
        est, det = self.est, self.est.detector
        qn = len(que_imgs)
        missing, extra = [n for n in self.names if n not in poses], sorted(set(poses) - set(self.names))
        if missing or extra:
            raise ValueError(f'verify_poses: need poses for exactly the set\'s objects {self.names}; missing {missing}, unknown {extra}')
        arrs = [np.asarray(poses[n]) for n in self.names]
        if qn == 0 or len(que_Ks) != qn or any(a.shape != (qn, 3, 4) for a in arrs):
            raise ValueError(f'verify_poses: {qn} frames, {len(que_Ks)} intrinsics and poses {[a.shape for a in arrs]}; need one K '
                             'and, per object, one pose [3,4] per frame, and at least one frame')
        if len({a.dtype for a in arrs}) != 1:
            raise ValueError('verify_poses: the objects\' poses have different dtypes; pass one dtype (float32: float32 values)')
        f32 = arrs[0].dtype == np.float32
        imgs = F.as_frames(que_imgs, 'verify_poses', det)
        if F.is_mixed(imgs):
            F.check_frames(imgs, que_Ks, 'verify_poses')
        nodes = self._verify_fn(key)
        with torch.no_grad():
            name, fn, fin = F.stage(det, ('verify_poses', int(f32)) + key, lambda u8, cams, p: nodes(u8, cams, p, f32), imgs)
            cams = det._to_dev(glue.cameras(np.stack([np.asarray(K) for K in que_Ks], 0)))
            p = det._to_dev(np.ascontiguousarray(np.concatenate(arrs, 0), np.float64).reshape(-1, 12))
            host = det._to_host(self.stages.run(name, fn, fin + [cams, p]))      # the call's one synchronising read
        res = verify.decode(host, len(arrs) * qn)
        return {name: {k: v[o * qn:(o + 1) * qn] for k, v in res.items()} for o, name in enumerate(self.names)}

    def tracker(self, num_sequences=1, refine_iter=1, smooth_num=5, smooth_std=2.5, bboxes=None, draw=None, draw_colors=None,
                verify_every=None, lost_score=None, lost_gate=None):
        """An ObjectTracker (gen6d_b200/track.py): every object of the set followed through `num_sequences` videos in
        lockstep, with Tracker's semantics per object; each step is one captured graph and one synchronising read.
        bboxes: {name: 8 box corners [8,3]}; a missing name takes the box of the object's database point cloud.
        draw / draw_colors {name: (R, G, B)}: every step also draws every object's box on its sequence's frame, as
        Gen6DEstimator.tracker(draw=) does (row f16).  verify_every, lost_score, lost_gate: as for
        Gen6DEstimator.tracker() (row f20), every object checked against its own references; a sequence is re-initialised
        if any of its objects is judged lost."""
        from .track import ObjectTracker
        return ObjectTracker(self, num_sequences, refine_iter=refine_iter, smooth_num=smooth_num, smooth_std=smooth_std,
                             bboxes=bboxes, draw=draw, draw_colors=draw_colors, verify_every=verify_every, lost_score=lost_score,
                             lost_gate=lost_gate)

    def instance_tracker(self, num_sequences=1, max_instances=4, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1,
                         min_score=None, nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5, bboxes=None, draw=None,
                         draw_colors=None, schedule='lockstep', verify_every=None, lost_score=None, lost_gate=None):
        """An ObjectInstanceTracker (gen6d_b200/instance_track.py): every instance of every object of the set, up to
        `max_instances` per object and frame, followed through `num_sequences` videos in lockstep, with
        Gen6DEstimator.instance_tracker()'s semantics per object (each object's tracks are matched only to its own
        detections) and track ids unique over the whole tracker.  Re-detection steps share the set's query pyramid and
        correlation; each step is one captured graph and one synchronising read.  bboxes, draw, draw_colors: as for
        tracker(); only live slots (track id >= 0) are drawn.
        schedule (row f18): 'lockstep' (every sequence re-detects on the same steps), 'per_sequence' (each sequence has its
        own re-detection flag and counter; reset / redetect take sequences, and step takes sequences= to step any subset)
        or 'staggered' ('per_sequence' with the periodic re-detections spread over the steps; needs redetect_every).
        verify_every, lost_score, lost_gate: as for Gen6DEstimator.instance_tracker() (row f21), each object's windows
        detected against its own references; a sequence re-detects when any slot of any object is judged lost."""
        from .instance_track import ObjectInstanceTracker
        return ObjectInstanceTracker(self, num_sequences, max_instances=max_instances, refine_iter=refine_iter,
                                     redetect_every=redetect_every, gate=gate, max_misses=max_misses, min_score=min_score,
                                     nms_iou=nms_iou, peak_radius=peak_radius, smooth_num=smooth_num, smooth_std=smooth_std,
                                     bboxes=bboxes, draw=draw, draw_colors=draw_colors, schedule=schedule,
                                     verify_every=verify_every, lost_score=lost_score, lost_gate=lost_gate)

    def raw_correlation(self, que_imgs):
        """The detector's raw correlation maps for inspection: {name: [scale][level] float32 [qn, H, W, rfn]} (the maps
        _detect_nhwc(return_taps=True)['raw'] holds for a single object), computed eagerly with the shared pyramid."""
        self._check()
        det = self.est.detector
        qn = len(que_imgs)
        with torch.no_grad():
            frames = det.upload_frame([np.asarray(f) for f in que_imgs])
            _, taps = self._detect(frames, return_taps=True)
        return {name: [[m[o * qn:(o + 1) * qn] for m in scale] for scale in taps['raw']]
                for o, name in enumerate(self._objects)}
