"""Drawn frames on the device (row f16): what drawing predict.py's smoothed box costs, on T frames rendered at 540x960
and upscaled once, before any timing, to 1080x1920 NV12 surfaces on the device.  One JSON line with the card and its power
limit read in the same run.

(a) draw node: g6d_draw_boxes alone, S working frames of 540x960 into NV12 destinations, CUDA events over --iters
    launches captured in one graph (median of --repeats runs); gb_s from shapes (one RGB read and one NV12 write per
    frame).
(b) est.tracker() and est.instance_tracker(max_instances=2) at each S, end to end over T steps, three feeds timed
    alternately, each reported as median [min, max] of --repeats runs, in sequence-frames/s:
      * plain: Resized(nv12, max_side=960) without drawing;
      * draw:  Resized(nv12, max_side=960), draw='smoothed' into S caller NV12 surfaces of 540x960 (out=);
      * host:  the workaround: each surface downloaded, cv2.cvtColor(COLOR_YUV2RGB_NV12) and cv2.resize to 540x960, the
               numpy tracker, then the box drawn with cv2 (draw_bbox_3d on the smoothed poses, every live slot for the
               instance tracker) and cv2.cvtColor(COLOR_RGB2YUV_I420).
    graph_kernels: C-ABI kernels per captured graph; peak_reserved_gb: torch.cuda.max_memory_reserved() over a capturing
    run of that feed alone (no other tracker alive, cache emptied and statistics reset before).
  python tools/draw_bench.py [--S 1,4,10] [--T 40] [--repeats 3]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='1,4,10')
    ap.add_argument('--T', type=int, default=40)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--iters', type=int, default=200)
    args = ap.parse_args()
    Ss = sorted({int(s) for s in args.S.split(',')})
    import cv2
    import numpy as np
    import torch
    from device_frames_bench import nv12_surface
    from gen6d_b200 import draw as dr, frames as fr, synthetic as syn
    from golden import track_cases
    from track_bench import card

    T, med = args.T, statistics.median
    db = syn.synthetic_database(height=540, width=960)
    est = syn.build_estimator(db)[0]
    est.cfg['device_glue'] = True
    K = db.K.astype(np.float64)
    up = lambda img: cv2.resize(img, (1920, 1080), interpolation=cv2.INTER_LINEAR)
    vids = [[nv12_surface(up(db.render(p, db.K))) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), T)]
            for s in range(max(Ss))]
    h, w = 540, 960

    def nv12_out(S):
        surf = [torch.empty(h * 3 // 2, w, dtype=torch.uint8, device='cuda') for _ in range(S)]
        return [fr.NV12(s[:h], s[h:]) for s in surf]

    E = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]

    def cv_draw(img, bbox, pose, K32):       # predict.py: draw_bbox_3d(img, project_points(bbox, pose, K), (0, 0, 255))
        p = bbox @ pose[:, :3].T + pose[:, 3:].T
        p = p @ K32.T
        d = p[:, 2]
        d[(np.abs(d) < 1e-4) & (np.abs(d) > 0)] = 1e-4
        q = np.round(p[:, :2] / d[:, None]).astype(np.int32)
        for c in q:
            cv2.circle(img, (int(c[0]), int(c[1])), 2, (255, 0, 0), -1)
        for a, b in E:
            img = cv2.line(img, (int(q[a][0]), int(q[a][1])), (int(q[b][0]), int(q[b][1])), (0, 0, 255), 2)
        return img

    K32 = K.astype(np.float32)
    res = {'tool': 'draw_bench', 'T': T, 'repeats': args.repeats, 'trackers': {}}
    makers = {'tracker': lambda S, **k: est.tracker(num_sequences=S, **k),
              'instance_tracker': lambda S, **k: est.instance_tracker(num_sequences=S, max_instances=2, **k)}
    for tname, make in makers.items():
        for S in Ss:
            outs = {'smoothed': nv12_out(S)}

            def run(name, tr):
                tr.reset()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for t in range(T):
                    if name == 'host':
                        work = []
                        for s in range(S):
                            f = vids[s][t]
                            yuv = torch.cat([f.y, f.uv], 0).cpu().numpy()
                            work.append(cv2.resize(cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12), (w, h), interpolation=cv2.INTER_LINEAR))
                        r = tr.step(work, [K] * S)
                        for s in range(S):
                            img = work[s]
                            if tname == 'tracker':
                                img = cv_draw(img, tr.bbox, r[1][s], K32)
                            else:
                                for m in range(r[2].shape[1]):
                                    if r[2][s, m] >= 0:
                                        img = cv_draw(img, tr.bbox, r[1][s, m], K32)
                            cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
                    else:
                        frames = [fr.Resized(vids[s][t], max_side=960) for s in range(S)]
                        tr.step(frames, [K] * S, **({'out': outs} if name == 'draw' else {}))
                torch.cuda.synchronize()
                return S * T / (time.perf_counter() - t0)

            kw = {'plain': {}, 'draw': {'draw': 'smoothed'}, 'host': {}}
            peak, kernels = {}, {}
            for name in kw:                      # each feed alone: its capturing run's peak memory
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                tr = make(S, **kw[name])
                run(name, tr)
                peak[name] = round(torch.cuda.max_memory_reserved() / 2 ** 30, 2)
                kernels[name] = sorted(st.kernels for st in tr.stages.stages.values())
                del tr
            trackers = {name: make(S, **kw[name]) for name in kw}
            for name, tr in trackers.items():
                run(name, tr)                    # capture
            rates = {n: [] for n in kw}
            for _ in range(args.repeats):
                for name, tr in trackers.items():
                    rates[name].append(run(name, tr))
            row = {'e2e_seq_frames_s': {n: [round(med(v), 1), round(min(v), 1), round(max(v), 1)] for n, v in rates.items()},
                   'graph_kernels': {n: kernels[n] for n in ('plain', 'draw')}, 'peak_reserved_gb': peak}
            if tname == 'tracker':               # (a) the draw node alone over S working frames
                drawer = trackers['draw']._drawer
                plan = fr.FramePlan([(h, w)] * S)
                table, _ = drawer.destinations(est.detector, plan, outs)
                frames_t = torch.randint(0, 256, (S, h, w, 3), dtype=torch.uint8, device='cuda')
                raw = torch.zeros(S, 12, dtype=torch.float64, device='cuda')
                smoothed = torch.from_numpy(np.tile(db.get_pose(str(11)).reshape(1, 12), (S, 1)).astype(np.float64)).cuda()
                Ks = torch.from_numpy(np.tile(K.reshape(1, 9), (S, 1))).cuda()
                node = lambda: drawer.node(est.detector, plan, frames_t, raw, True, smoothed, Ks, table)
                node()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for _ in range(args.iters):
                        node()
                times = []
                for _ in range(args.repeats):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    g.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1) / args.iters)
                us = med(times) * 1e3
                nbytes = S * (h * w * 3 + h * w * 3 // 2)
                row['draw_node'] = {'us': round(us, 2), 'gb_s': round(nbytes / (us * 1e-6) / 1e9, 1)}
                del g
            res['trackers'].setdefault(tname, {})[S] = row
            del trackers
            torch.cuda.empty_cache()
    res['card'], res['power_limit_w'] = card()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
