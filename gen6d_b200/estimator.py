"""Gen6DEstimator on the H100 networks: same constructor / build / predict contract as the
reference's estimator.py:94-216 (numpy images and poses in, numpy pose out; `ref_info`, `cfg`).

The stage sequencing is inherently serial per frame (crop depends on the detection, refinement
k+1 on pose k), so this class keeps the reference's structure; throughput comes from the kernels,
from keeping every reference-side tensor resident on the device, and from running independent
frames on independent GPUs (see gen6d_b200/dist.py).
"""
import os

import numpy as np
import torch
import yaml

from . import boxes as B
from . import frames as F
from . import geometry as G
from . import glue
from . import instances
from . import ops
from .graphs import StageCache
from .network import name2network


class Gen6DEstimator:
    default_cfg = {
        'ref_resolution': 128,
        'ref_view_num': 64,
        'det_ref_view_num': 32,
        'selector': None,
        'detector': None,
        'refiner': None,
        'refine_iter': 3,
        'device_build': False,    # True: cut the 64 + 5x64 reference crops of build() with the device warp kernel (row f2)
        'host_warps': False,      # True: keep the between-stage crops on the host in OpenCV, as the reference does
        'host_threads': None,     # OpenCV / torch-CPU threads for the host geometry (None: min(8, usable CPUs))
        # predict_batch / predict_many(batch > 1) keep the camera algebra between the stages on the device: the whole
        # batch prediction is ONE captured graph (csrc/glue.cu), no host round trips.  False (or G6D_DEVICE_GLUE=0):
        # the host sequences the stages with numpy geometry in between, as predict() does.
        'device_glue': os.environ.get('G6D_DEVICE_GLUE', '1') != '0',
    }

    def __init__(self, cfg, modules=None):
        """cfg: the reference's estimator yaml as a dict (configs/gen6d_pretrain.yaml).  `modules`
        optionally injects already-built networks {'detector','selector','refiner'} (used with
        synthetic checkpoints); otherwise they are loaded like estimator.py:117-125 does."""
        self.cfg = {**self.default_cfg, **cfg}
        self.ref_info = {}
        self.stages = StageCache()        # whole-prediction graphs of the device-glue path
        self._glue = None
        G.configure_host_threads(self.cfg['host_threads'])
        if modules is not None:
            self.detector, self.selector = modules['detector'], modules['selector']
            self.refiner = modules.get('refiner')
        else:
            self.detector = self._load_module(self.cfg['detector'])
            self.selector = self._load_module(self.cfg['selector'])
            self.refiner = self._load_module(self.cfg['refiner']) if self.cfg['refiner'] is not None else None

    @staticmethod
    def _load_module(cfg_path):
        with open(cfg_path, 'r') as f:
            cfg = yaml.load(f, Loader=yaml.FullLoader)
        net = name2network[cfg['network']](cfg)
        state = torch.load(f'data/model/{cfg["name"]}/model_best.pth', map_location='cpu')
        net.load_state_dict(state['network_state_dict'])
        print(f'load from {cfg["name"]}/model_best.pth step {state["step"]}')
        return net.cuda().eval()

    def build(self, database, split_type='all'):
        """estimator.py:139-171: pick 64 well-spread reference views, normalise them to 128x128
        look-at crops, make the 5 in-plane rotated copies, and load the three networks."""
        if split_type != 'all':
            raise NotImplementedError("only the 'all' split (reference ids = all database ids) is supported")
        from .database import as_object_database
        database = as_object_database(database)       # reference-repo databases are wrapped on the fly
        self._drop_workers()                           # clones made for a previous object are stale now
        v = self._reference_views(database)
        self.detector.load_ref_imgs(v['imgs'][:self.cfg['det_ref_view_num']])
        self.selector.load_ref_imgs(v['ref_imgs'], v['poses'], v['center'], v['vert'])
        self.ref_info = {k: v[k] for k in ('imgs', 'ref_imgs', 'Ks', 'poses', 'center', 'ref_ids')}
        if self.refiner is not None:
            self.refiner.load_ref_imgs(database, v['ids_all'])
        torch.cuda.current_stream().synchronize()      # reference state complete before any other stream reads it

    def _reference_views(self, database):
        """The object-specific part of build(): FPS reference views, their normalised crops and rotated copies."""
        center, vert = database.object_center(), database.object_vert()
        ids_all = database.get_img_ids()
        ref_ids = G.select_views_fps(database, ids_all, self.cfg['ref_view_num'])
        res = self.cfg['ref_resolution']
        on_device = self.cfg['device_build']
        ref_imgs, ref_Ks, ref_poses, ref_Hs = G.normalize_reference_views(database, ref_ids, res, 0.05, warp=not on_device)
        rot_Hs = [[G.similarity_2d((res / 2, res / 2), 1.0, ang, (res / 2, res / 2)).astype(np.float32) @ ref_Hs[k]
                   for k in range(len(ref_ids))] for ang in (-np.pi / 2, -np.pi / 4, 0, np.pi / 4, np.pi / 2)]
        if on_device:
            # same bytes as the OpenCV path (g6d_warp_perspective_u8 is bit-exact), one launch per set
            srcs = [torch.from_numpy(np.ascontiguousarray(database.get_image(i))).to(self.detector.device) for i in ref_ids]
            cut = lambda Hs: ops.warp_perspective_u8(
                torch.from_numpy(G.pack_warp_jobs(srcs, [G.perspective_dst_to_src(H) for H in Hs])).to(srcs[0].device),
                len(srcs), res, res).cpu().numpy()
            ref_imgs = cut(list(ref_Hs))
            rots = [cut(Hs) for Hs in rot_Hs]
        else:
            import cv2
            rots = [np.stack([cv2.warpPerspective(database.get_image(i), Hs[k], (res, res), flags=cv2.INTER_LINEAR)
                              for k, i in enumerate(ref_ids)], 0) for Hs in rot_Hs]
        ref_imgs_rots = np.stack(rots, 0)  # an,rfn,h,w,3
        return {'imgs': ref_imgs, 'ref_imgs': ref_imgs_rots, 'Ks': ref_Ks, 'poses': ref_poses, 'center': center,
                'ref_ids': ref_ids, 'vert': vert, 'ids_all': ids_all}

    def predict(self, que_img, que_K, pose_init=None):
        """estimator.py:173-216.  que_img uint8 [h,w,3], que_K [3,3] -> (pose [3,4], inter_results).  A numpy frame only:
        frames on the GPU go through predict_batch (TypeError)."""
        F.host_only([que_img], 'predict()')
        inter = {}
        res = self.cfg['ref_resolution']
        host_warps = self.cfg['host_warps']
        # the frame goes to the device once; the detection crop and the refinement look-at crops are
        # cut from it there (bit-exact with the OpenCV warps the reference runs on the host)
        frame = None if host_warps else self.detector.upload_frame(que_img)
        if pose_init is None:
            det = self.detector.detect_que_imgs(que_img[None], que_dev=None if host_warps else frame[None])
            position, scale_r2q = det['positions'][0], det['scales'][0]
            if host_warps:
                crop, _ = G.crop_similarity(que_img, position, 1 / scale_r2q, 0, res)
                sel = self.selector.select_que_imgs(crop[None])
            else:
                _, M = G.crop_similarity(None, position, 1 / scale_r2q, 0, res)
                sel = self.selector.select_from_frame(frame, M, res)
                crop = sel['que_imgs'][0]
            inter.update(det_position=position, det_scale_r2q=scale_r2q, det_que_img=crop)
            ref_idx, angle_r2q, scores = sel['ref_idx'][0], sel['angles'][0], sel['scores'][0]
            inter.update(sel_angle_r2q=angle_r2q, sel_scores=scores, sel_ref_idx=ref_idx)
            pose = G.pose_from_similarity(position, scale_r2q, angle_r2q, self.ref_info['poses'][ref_idx],
                                          self.ref_info['Ks'][ref_idx], que_K, self.ref_info['center'])
        else:
            pose = pose_init
        if self.refiner is not None:
            poses = [pose]
            for _ in range(self.cfg['refine_iter']):
                pose = self.refiner.refine_que_imgs(que_img, que_K, pose, size=128, ref_num=6, ref_even=True,
                                                    que_dev=frame, host_warps=host_warps)
                poses.append(pose)
            inter['refine_poses'] = poses
        return pose, inter


    def predict_batch(self, que_imgs, que_Ks, pose_inits=None, boxes=None):
        """predict() for a batch of independent frames (row f3): qn frames go through ONE
        detect stage, ONE select stage and ONE refine stage per iteration -- 2 + refine_iter graph launches
        and device->host reads for the whole batch instead of per frame -- with the small per-frame camera
        algebra on the host in between.  Same results as predict() frame by frame.  Frames of different sizes take the
        device-glue path only (row f13: detection per size, the crops cut from one zero-padded canvas).
        que_imgs: list / array of uint8 [h,w,3]; que_Ks: [qn,3,3].  Returns (poses [qn,3,4], inter dict of lists).
        On the device-glue path que_imgs may instead be device frames (row f14; frames.as_frames): CUDA uint8 RGB tensors
        [h,w,3] with any row pitch (or one [qn,h,w,3] tensor) and frames.NV12 decoder surfaces, mixed freely, with the
        numpy path's results on the same RGB bytes.  They must be ready on the current stream; the call ends in its
        synchronising read, after which they may be overwritten or freed.

        boxes (row f19): the object's box on every frame from another detector, exactly one per frame ([4] x0, y0, x1, y1
        or [5] with a score, or [1, 4|5]; numpy or CUDA float32, in the frame's pixels; gen6d_b200/boxes.py).  The
        detector does not run: the call is predict_instances(max_instances=1, boxes=) with its [:, 0] rows, and inter
        also holds 'det_score' [qn], the box scores.  Needs the device pipeline, and pose_inits None.  Numpy boxes are
        checked on the host (ValueError when non-finite or degenerate); a CUDA box is not read, and one that is not
        usable gives the empty detection record (position (0, 0), scale 1, det_score -inf), whose pose is meaningless."""
        if boxes is not None:
            return self._predict_batch_boxes(que_imgs, que_Ks, pose_inits, boxes)
        qn, res = len(que_imgs), self.cfg['ref_resolution']
        que_Ks = [np.asarray(K) for K in que_Ks]
        device = self.cfg['device_glue'] and pose_inits is None and self._glue_possible()
        imgs = F.as_frames(que_imgs, 'predict_batch', self.detector,
                           None if device else "predict_batch with pose_inits, cfg['device_glue'] off or cfg['host_warps'] on")
        if F.is_device(imgs):                        # frames already on the GPU: gathered in the graph (row f14)
            return self._predict_batch_device(None, que_Ks, F.check_frames(imgs, que_Ks, 'predict_batch'))
        if F.is_mixed(imgs):                         # frames of different sizes: the device glue path only (row f13)
            if not device:
                F.require_one_size(imgs, "predict_batch with pose_inits, cfg['device_glue'] off or cfg['host_warps'] on")
            return self._predict_batch_device(None, que_Ks, F.check_frames(imgs, que_Ks, 'predict_batch'))
        frames = self.detector.upload_frame(imgs)  # [qn,h,w,3] once, for all stages
        if device:
            return self._predict_batch_device(frames, que_Ks)
        inter = {}
        if pose_inits is None:
            det = self.detector.detect_que_imgs(None, que_dev=frames)
            Ms = [G.crop_similarity(None, det['positions'][i], 1 / det['scales'][i], 0, res)[1] for i in range(qn)]
            sel = self.selector.select_from_frames(frames, Ms, res)
            inter.update(det_position=det['positions'], det_scale_r2q=det['scales'], det_que_img=sel['que_imgs'],
                         sel_angle_r2q=sel['angles'], sel_scores=sel['scores'], sel_ref_idx=sel['ref_idx'])
            ridx = np.asarray(sel['ref_idx'])
            poses = G.poses_from_similarity(det['positions'], det['scales'], sel['angles'], self.ref_info['poses'][ridx],
                                            self.ref_info['Ks'][ridx], np.stack(que_Ks, 0), self.ref_info['center'])
        else:
            poses = np.stack(pose_inits, 0)
        if self.refiner is not None:
            poses, inter['refine_poses'] = self._refine_batch_host(frames, que_Ks, poses, self.cfg['refine_iter'])
        return poses, inter

    def _predict_batch_boxes(self, que_imgs, que_Ks, pose_inits, boxes):
        """predict_batch(boxes=): predict_instances(max_instances=1, boxes=) in predict_batch's return contract."""
        from .objects import require_device_pipeline
        require_device_pipeline(self, 'predict_batch(boxes=)')
        if pose_inits is not None:
            raise ValueError('predict_batch: boxes= detects the initial poses; pass boxes or pose_inits, not both')
        poses, inter = self.predict_instances(que_imgs, que_Ks, max_instances=1,
                                              boxes=B.one_per_frame(boxes, len(que_imgs), 'predict_batch'))
        keys = ('det_position', 'det_scale_r2q', 'det_score', 'det_que_img', 'sel_angle_r2q', 'sel_scores', 'sel_ref_idx')
        one = {k: np.ascontiguousarray(inter[k][:, 0]) for k in keys}
        one['refine_poses'] = [np.ascontiguousarray(c[:, 0]) for c in inter['refine_poses']]
        return np.ascontiguousarray(poses[:, 0]), one

    def _refine_batch_host(self, frames, que_Ks, poses, iters):
        """`iters` host-sequenced batched refinements from poses [qn,3,4] -> (poses, [poses, refined 1, ..., refined iters])."""
        chain = [poses]
        for _ in range(iters):
            poses = self.refiner.refine_batch(frames, que_Ks, poses, size=128, ref_num=6, ref_even=True)
            chain.append(poses)
        return poses, chain

    # ------------------------------------------------------------------ device-resident prediction
    def _glue_possible(self):
        return self.refiner is not None and getattr(self.selector.comm, 'capturable', False) and not self.cfg['host_warps']

    def _glue_state(self):
        """Device tables of the camera algebra (glue.py), rebuilt when any module's state changed."""
        gen = self._generation()
        if self._glue is None or self._glue['gen'] != gen:
            self._glue = {'gen': gen, **self._device_tables(self.ref_info, self.refiner.refs)}
            self.stages.clear()
        return self._glue

    def _device_tables(self, ref_info, refiner_refs):
        """Device copies of one object's glue tables (selector references from `ref_info`, the refiner's views and
        resident images from `refiner_refs`) and the g6d_glue_refs / g6d_glue_views structs pointing at them."""
        dev = self.detector.device
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        refs = glue.selector_refs(ref_info)
        refs_dev = {k: up(refs[k]) for k in ('poses', 'cen', 'f', 'dist')}
        tables = glue.refiner_views(refiner_refs.database, refiner_refs.ids, 128, 6)
        src = self.refiner._ref_sources(refiner_refs.ids, refiner_refs)
        views_dev = {k: up(tables[k]) for k in ('poses', 'R_look', 'RlookR', 'f', 'Kinv', 'even_idx', 'even_dirs')}
        views_dev['src'] = up(np.asarray([s[0] for s in src], np.uint64).view(np.int64))
        views_dev['rows'], views_dev['cols'] = up(np.asarray([s[1] for s in src], np.int32)), up(np.asarray([s[2] for s in src], np.int32))
        torch.cuda.current_stream().synchronize()
        ptr = lambda d: {k: t.data_ptr() for k, t in d.items()}
        return {'keep': (refs_dev, views_dev), 'tables': tables,
                'refs': glue.refs_struct({**ptr(refs_dev), 'center': refs['center']}),
                'views': glue.views_struct(ptr(views_dev), tables, views_dev['src'].data_ptr(), views_dev['rows'].data_ptr(),
                                           views_dev['cols'].data_ptr())}

    def _initial_poses_device_fn(self, st, detect=None):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> detection, selection and the initial poses float64 [M*qn,12]:
        (poses, det, crop, idx, sel_out, logits), enqueued back to back.  detect(frames) -> det [M*qn,4] (x, y, scale,
        score; row m*qn + f is instance m on frame f) is the detection step: the score-map argmax (M = 1) by default,
        _peaks_detect_fn's instances for predict_instances.  Every instance slice gets its own crop jobs and initial
        poses; the M*qn crops go through one warp and one selection."""
        res = self.cfg['ref_resolution']
        select = self.selector._select_warped(res)
        detect = detect or (lambda u8: F.per_size(self.detector._detect_u8, u8))      # once per frame size (row f13)

        def fn(frames, cams):
            qn = frames.shape[0]
            det = detect(frames)
            sl = [slice(m * qn, (m + 1) * qn) for m in range(det.shape[0] // qn)]
            jobs = [ops.glue_detection_jobs(det[s], frames, res) for s in sl]
            crop, idx, sel_out, logits = select(jobs[0] if len(sl) == 1 else torch.cat(jobs))
            poses = [ops.glue_initial_poses(det[s], idx[s], sel_out[s], st['refs'], cams) for s in sl]
            return (poses[0] if len(sl) == 1 else torch.cat(poses)), det, crop, idx, sel_out, logits
        return fn

    def _peaks_detect_fn(self, max_instances, peak_radius, nms_iou, min_score):
        """frames u8 [qn,h,w,3] -> (det [M*qn,4] instance-major, valid int32 [M*qn], count int32 [qn]): the detector's maps
        and g6d_det_parse_peaks.  `extra` receives valid and count when the returned function runs."""
        det_mod, box = self.detector, float(self.cfg['ref_resolution'])
        extra = []

        def one_size(u8):
            o = det_mod._detect_nhwc(ops.preprocess_u8(u8, out_c=3, imagenet_norm=False))
            det, _, valid, count = ops.det_parse_peaks(o['score_predict'], o['scale_predict'], o['offset_predict'], max_instances,
                                                       peak_radius, nms_iou, box, min_score, det_mod.pool_ratio)
            return det.reshape(-1, 4), valid.reshape(-1), count

        def detect(frames):
            det, valid, count = F.per_size(one_size, frames)                       # once per frame size (row f13)
            extra[:] = [valid, count]
            return det
        return detect, extra

    def _predict_device_fn(self, st):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> every stage of predict_batch, enqueued back to back."""
        iters, R = self.cfg['refine_iter'], st['tables']['ref_num']
        initial, refine = self._initial_poses_device_fn(st), self.refiner._refine_warped(128)

        def fn(frames, cams):
            poses, det, crop, idx, sel_out, logits = initial(frames, cams)
            chain = [poses]
            for it in range(iters):
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems(st['views'], R, cams, frames, poses, it > 0)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)
                poses = ops.glue_apply_refinements(st['views'], que_pose, que_K, rect, out)
                chain.append(poses)
            return torch.stack(chain, 0), det, crop, idx, sel_out, logits
        return fn

    def _predict_batch_device(self, frames, que_Ks, imgs=None):
        """predict_batch with cfg['device_glue']: one graph launch, one synchronising read at the end.  imgs: frames of
        different sizes (numpy, not uploaded; frames is None), packed and put on a canvas in the graph."""
        st = self._glue_state()
        qn = len(que_Ks)
        with torch.no_grad():
            if imgs is None:
                name, fn, fin = 'predict', self._predict_device_fn(st), [frames]
            else:
                name, fn, fin = F.stage(self.detector, 'predict', self._predict_device_fn(st), imgs)
            cams = self.detector._to_dev(glue.cameras(np.stack(que_Ks, 0)))
            outs = self.stages.run(name, fn, fin + [cams])
            chain, det, crop, idx, sel_out, logits = [self.detector._to_host(t) for t in outs]
        chain = chain.reshape(len(chain), qn, 3, 4)
        poses0, refined = chain[0], [c.astype(np.float32) for c in chain[1:]]
        inter = {'det_position': det[:, :2].copy(), 'det_scale_r2q': det[:, 2].copy(), 'det_que_img': crop,
                 'sel_angle_r2q': sel_out[:, 0].copy(), 'sel_scores': logits, 'sel_ref_idx': idx,
                 'refine_poses': [poses0] + refined}
        return (refined[-1] if refined else poses0), inter

    # ------------------------------------------------------------------ several instances per frame (instances.py)
    def _instances_fn(self, st, M, radius, nms_iou, min_score, boxes=None):
        """frames u8 [qn,h,w,3], cams f64 [qn,20] -> packed results of predict_instances: the detector's maps, the peaks,
        M*qn crops and selections, and refine_iter x (glue over M slots, ONE refiner stage over M*qn poses, glue).
        boxes: a boxes.Detect, the detection step from caller boxes instead of the maps and peaks."""
        iters, R = self.cfg['refine_iter'], st['tables']['ref_num']
        detect, extra = (boxes, boxes.extra) if boxes is not None else self._peaks_detect_fn(M, radius, nms_iou, min_score)
        initial, refine = self._initial_poses_device_fn(st, detect), self.refiner._refine_warped(128)
        views = [st['views']] * M

        def fn(frames, cams):
            poses, det, crop, idx, sel_out, logits = initial(frames, cams)
            chain = [poses]
            for it in range(iters):
                jobs, que_K, que_pose, rect, ref_Ks, ref_poses, _ = ops.glue_refine_problems_objects(views, R, cams, frames, poses, it > 0)
                out = refine(jobs, que_K, que_pose, ref_Ks, ref_poses)
                poses = ops.glue_apply_refinements_objects(views, que_pose, que_K, rect, out)
                chain.append(poses)
            return instances.pack([torch.stack(chain, 0), det, idx, sel_out, logits] + extra, crop)
        return fn

    def predict_instances(self, que_imgs, que_Ks, max_instances=4, min_score=None, nms_iou=0.3, peak_radius=1, boxes=None):
        """Every instance of the object on qn frames (of one size or several, row f13): up to `max_instances` detections per frame, the peaks of
        the detector's score map (within `peak_radius` cells) kept by greedy non-maximum suppression of their
        ref_resolution * scale boxes at IoU > `nms_iou` (g6d_det_parse_peaks), each selected and refined as predict_batch
        does.  min_score: a raw score-head threshold (its meaning depends on the checkpoint); None: no threshold.
        Returns (poses float32 [qn,M,3,4], inter): predict_batch's device-glue keys led by [qn, M], 'det_score' [qn,M],
        'refine_poses' a list of [qn,M,3,4], 'instance_valid' bool [qn,M] and 'instance_count' [qn].  Instance 0 is
        predict_batch's detection.  Rows of instances that were not found are computed too (on a repeat of instance 0's
        detection, so the graph keeps its shapes) and returned, masked by instance_valid: use only the valid rows.
        One captured graph per (qn, frame shape, max_instances, peak_radius, nms_iou, min_score), one read per call.
        que_imgs may be device frames, with predict_batch's rules (row f14).

        boxes (row f19): the instances from another detector instead of the score map, one entry per frame: a numpy array
        or CUDA float32 tensor [n, 4] (x0, y0, x1, y1) or [n, 5] (with a score), n >= 0, in the frame's pixels (a Resized
        frame's working pixels); gen6d_b200/boxes.py.  The detector runs no kernel: g6d_det_from_boxes makes instance m
        of a frame its m-th usable box by score (the square on the box's longer side, so scale = side / ref_resolution),
        at most max_instances, and everything after the detection is unchanged.  det_score holds the box scores (0 for
        [n, 4]), instance_valid / instance_count the boxes kept.  min_score, nms_iou and peak_radius do not apply to boxes
        (the caller's detector thresholds and suppresses) and are not part of the box graphs' key: one graph per (qn,
        frame shape, max_instances, box bucket N), N the next power of two of the longest list.  CUDA boxes must be
        ready on the current stream."""
        from .objects import require_device_pipeline
        require_device_pipeline(self, 'predict_instances')
        key = instances.check_args(max_instances, nms_iou, peak_radius, min_score)
        M = key[0]
        qn, res = len(que_imgs), self.cfg['ref_resolution']
        if qn == 0 or len(que_Ks) != qn:
            raise ValueError(f'predict_instances: {qn} frames and {len(que_Ks)} intrinsics; need one K per frame and at least one frame')
        imgs = F.as_frames(que_imgs, 'predict_instances', self.detector)
        if F.is_mixed(imgs):
            F.check_frames(imgs, que_Ks, 'predict_instances')
        table = None if boxes is None else B.for_frames(boxes, qn, 'predict_instances', self.detector.device)
        st = self._glue_state()
        det = self.detector
        with torch.no_grad():
            if table is None:
                name, fn, tail = ('instances',) + key, self._instances_fn(st, *key), []
            else:
                dt = B.Detect(M, 1, qn, table.N, B.inv_box_size(res))
                name, fn = B.graph_name(('instances', M), table.N), dt.bind(self._instances_fn(st, *key, boxes=dt))
                tail = [table.upload(det)]
            name, fn, fin = F.stage(det, name, fn, imgs)
            cams = det._to_dev(glue.cameras(np.stack([np.asarray(K) for K in que_Ks], 0)))
            buf = self.stages.run(name, fn, fin + [cams] + tail)
            host = det._to_host(buf)                                       # the call's one synchronising read
        n, n_sel = M * qn, len(self.ref_info['poses'])
        rd = instances.Unpacker(host, n * res * res * 3)
        chain = rd.take((self.cfg['refine_iter'] + 1) * n * 12).reshape(-1, n, 12)
        parts = [rd.take(n * 4), rd.take(n), rd.take(n * 2), rd.take(n * n_sel), rd.take(n), rd.take(qn)]
        return instances.inter_of(chain, *parts, rd.crops.reshape(n, res, res, 3), M, qn)

    # ------------------------------------------------------------------ checking poses with the detector (row f20)
    def _verify_fn(self, st, key, M=1):
        """The verification nodes (verify.nodes) of this estimator's object; M: row groups (an instance tracker's slots)."""
        from . import verify
        return verify.nodes(self, [st['refs']], [self.detector._detect_u8], key, M)

    def verify_poses(self, frames, Ks, poses, lost_score=None, lost_gate=None):
        """Check each pose with the detector on a window around the object (row f20; gen6d_b200/verify.py).  Pose i on
        frame i (predict_batch's frame forms: numpy, of one size or several, CUDA RGB, frames.NV12, frames.Resized; Ks
        [n,3,3]; poses [n,3,4], a float32 array read as float32 values, any other dtype as float64) becomes the detection
        record that would have produced it: its projected object centre and scale.  A 2 x ref_resolution window is cut
        there (the object at its reference size in the middle), the detector runs on the windows, and its detection is
        mapped back to the frame.  Returns {'position' [n,2], 'scale' [n], 'score' [n] (the detector's raw score head),
        'offset' [n] (|position - projected centre| / (ref_resolution * window_scale)), 'lost' bool [n], 'window_center'
        [n,2], 'window_scale' [n]}.  lost: the pose's centre is not in front of the camera (or not finite), score <
        lost_score (NaN is lost) or offset > lost_gate; a threshold of None is not applied.  The thresholds' meaning
        depends on the checkpoint.  One captured graph per (n, frame pattern, pose dtype, thresholds), one read."""
        from . import verify
        from .objects import require_device_pipeline
        require_device_pipeline(self, 'verify_poses')
        key = verify.check_thresholds(lost_score, lost_gate)
        poses = np.asarray(poses)
        n = len(frames)
        if n == 0 or len(Ks) != n or poses.shape != (n, 3, 4):
            raise ValueError(f'verify_poses: {n} frames, {len(Ks)} intrinsics and poses {poses.shape}; need one K and one pose '
                             '[3,4] per frame and at least one frame')
        f32 = poses.dtype == np.float32
        imgs = F.as_frames(frames, 'verify_poses', self.detector)
        if F.is_mixed(imgs):
            F.check_frames(imgs, Ks, 'verify_poses')
        st = self._glue_state()
        det = self.detector
        nodes = self._verify_fn(st, key)
        with torch.no_grad():
            name, fn, fin = F.stage(det, ('verify_poses', int(f32)) + key, lambda u8, cams, p: nodes(u8, cams, p, f32), imgs)
            cams = det._to_dev(glue.cameras(np.stack([np.asarray(K) for K in Ks], 0)))
            p = det._to_dev(np.ascontiguousarray(poses, np.float64).reshape(n, 12))
            host = det._to_host(self.stages.run(name, fn, fin + [cams, p]))      # the call's one synchronising read
        return verify.decode(host, n)

    # ------------------------------------------------------------------ video tracking (predict.py)
    def tracker(self, num_sequences=1, refine_iter=1, smooth_num=5, smooth_std=2.5, bbox_3d=None, draw=None, draw_color=(0, 0, 255),
                verify_every=None, lost_score=None, lost_gate=None):
        """A Tracker for `num_sequences` videos stepped in lockstep (gen6d_b200/track.py): the first step is a full
        prediction with cfg['refine_iter'] refinements, every later step `refine_iter` refinements from the previous
        frame's pose, each followed by predict.py's box smoothing (`smooth_num` frames, `smooth_std`; defaults of
        predict.py's --num / --std).  bbox_3d: the object's 8 box corners [8,3]; None: from the database's point cloud.
        draw: 'raw', 'smoothed' or ('raw', 'smoothed'): every step also draws predict.py's images_out /
        images_out_smooth frames on the device, the box edges in draw_color (R, G, B) (Tracker.step, row f16).
        cfg['refine_iter'] is left untouched.  To start from another detector's boxes, pose the first frames with
        predict_batch(boxes=) and pass those poses to the tracker's start(poses, sequences).
        verify_every (row f20; needs the device pipeline): a refine step in which a stepped sequence has taken
        verify_every refine steps since its last full prediction, start(), reset() or verification also checks every
        stepped sequence's final pose as verify_poses(lost_score, lost_gate) does, inside the step's graph, and returns
        the result as inter['verify']; every sequence judged lost is then re-initialised as reset([s]) does.  Thresholds
        None: verify and report, never reset."""
        from .track import Tracker
        return Tracker(self, num_sequences, refine_iter=refine_iter, smooth_num=smooth_num, smooth_std=smooth_std,
                       bbox_3d=bbox_3d, draw=draw, draw_color=draw_color, verify_every=verify_every, lost_score=lost_score,
                       lost_gate=lost_gate)

    def instance_tracker(self, num_sequences=1, max_instances=4, refine_iter=1, redetect_every=None, gate=0.5, max_misses=1,
                         min_score=None, nms_iou=0.3, peak_radius=1, smooth_num=5, smooth_std=2.5, bbox_3d=None, draw=None,
                         draw_color=(0, 0, 255), schedule='lockstep', verify_every=None, lost_score=None, lost_gate=None):
        """An InstanceTracker (gen6d_b200/instance_track.py): every instance of the object, up to `max_instances` per frame,
        followed through `num_sequences` videos in lockstep.  The first step (and the one after reset() / redetect(), and
        every `redetect_every`-th step after the last re-detection) detects predict_instances' instances (min_score,
        nms_iou, peak_radius) and associates them with the live tracks: the greedy matching of the smallest
        |projected object centre - detected position| / (ref_resolution * detected scale) below `gate`; a track unmatched
        more than `max_misses` re-detections in a row is dropped, and unmatched detections start new tracks.  Every other
        step refines each track `refine_iter` times from its previous pose.  Both smooth as tracker() does.  draw /
        draw_color: as for tracker(); every live slot (track id >= 0) is drawn, in slot order.
        schedule (row f18): 'lockstep' (every sequence re-detects on the same steps), 'per_sequence' (each sequence has its
        own re-detection flag and counter; reset / redetect take sequences, and step takes sequences= to step any subset)
        or 'staggered' ('per_sequence' with the periodic re-detections spread over the steps; needs redetect_every).
        verify_every (row f21): a step in which a stepped sequence that does not re-detect has taken verify_every steps
        since its last re-detection, reset(), redetect() or verification also checks the final pose of every slot of
        every such sequence as verify_poses(lost_score, lost_gate) does, inside the step's graph, and returns the result
        as inter['verify'] ([S, M] per key; empty slots and re-detecting sequences NaN / not lost).  With a threshold, a
        live track judged lost takes a miss and is dropped past max_misses as an unmatched track is at a re-detection
        (inter['verify']['dropped'] lists the ids), one judged found restarts its misses, and every sequence with a lost
        track re-detects on its next step (detecting(); lockstep: every sequence).  Thresholds None: verify and report,
        never change a track."""
        from .instance_track import InstanceTracker
        return InstanceTracker(self, num_sequences, max_instances=max_instances, refine_iter=refine_iter,
                               redetect_every=redetect_every, gate=gate, max_misses=max_misses, min_score=min_score, nms_iou=nms_iou,
                               peak_radius=peak_radius, smooth_num=smooth_num, smooth_std=smooth_std, bbox_3d=bbox_3d,
                               draw=draw, draw_color=draw_color, schedule=schedule, verify_every=verify_every,
                               lost_score=lost_score, lost_gate=lost_gate)

    def track(self, que_imgs, que_K, **tracker_kwargs):
        """predict.py's loop over one video: que_imgs uint8 [h,w,3] frames of one size, que_K [3,3] (or one per frame).
        Returns [(pose, smoothed_pose, inter)] per frame: the raw pose [3,4], the smoothed pose [3,4] (float64, as
        pose_utils.pnp returns it) and that frame's intermediate results."""
        trk = self.tracker(num_sequences=1, **tracker_kwargs)
        Ks = np.asarray(que_K)
        out = []
        for t, img in enumerate(que_imgs):
            K = Ks[t] if Ks.ndim == 3 else Ks
            poses, smoothed, inter = trk.step([img], [K])
            one = {k: ([p[0] for p in v] if k == 'refine_poses' else v[0]) for k, v in inter.items()}
            out.append((poses[0], smoothed[0], one))
        return out

    # ------------------------------------------------------------------ several objects (gen6d_b200/objects.py)
    def object_set(self):
        """An ObjectSet over this estimator's networks (weights shared, loaded once): objects are added with their own
        reference state, and ObjectSet.predict poses every object on the same frames in one captured graph.  The
        estimator's own object (build) and the set's objects never affect each other."""
        from .objects import ObjectSet
        return ObjectSet(self)

    # ------------------------------------------------------------------ throughput API
    def worker_clone(self):
        import copy
        other = copy.copy(self)
        other._workers, other._pool, other._workers_gen = None, None, None
        other.stages = StageCache()                   # private graphs; the glue tables (self._glue) are shared, read-only
        other.detector, other.selector = self.detector.worker_clone(), self.selector.worker_clone()
        other.refiner = self.refiner.worker_clone() if self.refiner is not None else None
        return other

    def _generation(self):
        mods = (self.detector, self.selector, self.refiner)
        return tuple(m.generation for m in mods if m is not None)

    def _weights_generation(self):
        mods = (self.detector, self.selector, self.refiner)
        return tuple(m.weights_generation for m in mods if m is not None)

    def _drop_workers(self):
        pool = getattr(self, '_pool', None)
        if pool is not None:
            pool.shutdown(wait=True)
        self._workers, self._pool, self._workers_gen, self._warm = None, None, None, set()

    def predict_many(self, que_imgs, que_Ks, workers=2, batch=1):
        """Poses for independent frames: `workers` host threads, each with a clone of the networks (shared
        weights / reference features, private CUDA graphs) and a CUDA stream, each pushing `batch` frames
        at a time through predict_batch (batch = 1: plain predict), so one batch's host geometry overlaps
        another batch's kernels.  Same results as predict(); returns [(pose, inter)] (inter of a batched
        frame holds that frame's slices).  With batch > 1 the frames are grouped by size (in order of first
        appearance) before they are cut into batches, so every batch has frames of one size.  Numpy frames only (TypeError
        for frames on the GPU: predict_batch takes them)."""
        from concurrent.futures import ThreadPoolExecutor
        F.host_only(que_imgs, 'predict_many')
        if len(que_imgs) == 0:
            return []
        # The clones share weights / reference features by reference and own captured graphs over them:
        # rebuild them whenever any module's state changed (build() on another object, load_state_dict).
        if getattr(self, '_workers', None) is None or len(self._workers) != workers or self._workers_gen != self._generation():
            self._drop_workers()
            self._workers = [(self.worker_clone(), torch.cuda.Stream()) for _ in range(workers)]
            self._workers_gen = self._generation()
            self._pool = ThreadPoolExecutor(workers)
            self._warm = set()
        n = len(que_imgs)
        batch = max(1, min(batch, n))
        # batches are cut per frame size (groups in order of first appearance, input order inside a group), so every
        # batch is one predict_batch graph of one size
        sizes = F.size_pattern(que_imgs) if batch > 1 else [None] * n
        groups = [[i for i in range(n) if sizes[i] == z] for z in dict.fromkeys(sizes)]
        for g in groups:
            warm_key = (batch, bool(self.cfg['device_glue'])) + ((sizes[g[0]],) if len(groups) > 1 else ())
            if warm_key in self._warm:
                continue
            for est, stream in self._workers:        # capture every worker's graphs for this batch size / path, one at a time
                stream.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(stream):
                    if batch == 1:
                        est.predict(que_imgs[0], que_Ks[0])
                    else:
                        m = len(g)
                        est.predict_batch([que_imgs[g[i % m]] for i in range(batch)], [que_Ks[g[i % m]] for i in range(batch)])
                    stream.synchronize()
            self._warm.add(warm_key)
        results = [None] * n
        caller = torch.cuda.current_stream()
        chunks = [g[b:b + batch] for g in groups for b in range(0, len(g), batch)]

        def run(w):
            est, stream = self._workers[w]
            stream.wait_stream(caller)               # order after whatever the caller enqueued (uploads, a rebuild)
            with torch.cuda.stream(stream):
                for c in range(w, len(chunks), workers):
                    idx = chunks[c]
                    if batch == 1:
                        results[idx[0]] = est.predict(que_imgs[idx[0]], que_Ks[idx[0]])
                        continue
                    pad = idx + [idx[-1]] * (batch - len(idx))        # a short last chunk reuses the captured batch size
                    poses, inter = est.predict_batch([que_imgs[i] for i in pad], [que_Ks[i] for i in pad])
                    for j, i in enumerate(idx):
                        one = {k: ([p[j] for p in v] if k == 'refine_poses' else v[j]) for k, v in inter.items()}
                        results[i] = (poses[j], one)
                stream.synchronize()

        import sys
        old_si = sys.getswitchinterval()
        sys.setswitchinterval(2e-4)      # a worker that just got its D2H result should not wait 5 ms for the GIL
        try:
            list(self._pool.map(run, range(workers)))
        finally:
            sys.setswitchinterval(old_si)
        return results


name2estimator = {'gen6d': Gen6DEstimator}
