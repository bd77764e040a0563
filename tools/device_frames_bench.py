"""Frames already on the GPU (row f14): what device-frame input buys over numpy input, on tools/track_bench.py's and
tools/instance_track_bench.py's frames (T frames of 480x640, cfg['refine_iter'] = 3, tracker refine_iter = 1).  One JSON
line with the card and its power limit read in the same run.  For est.tracker() and est.instance_tracker(max_instances=2)
at each S, and predict_batch on 10 frames, four inputs timed alternately, each the median of --repeats runs:
  * dev:   device-resident, the numpy path's captured graphs replayed on frames already uploaded (no input, no read);
  * numpy: numpy frames end to end (the pinned staging copy and upload, one replay, one read, unpacking);
  * rgb:   CUDA uint8 [h,w,3] tensors end to end (the device-frame graph: table upload, g6d_frames_gather, the body);
  * nv12:  frames.NV12 surfaces end to end (the gather converts them).
Rates are sequence-frames/s (S frames per tracker step; qn frames per predict_batch call).  gather_us: g6d_frames_gather
alone for one step's frames (CUDA events over --gather-iters launches), and gather_mb its bytes moved, computed from
shapes (RGB reads 3 B/px, NV12 1.5 B/px; both write 3 B/px).
  python tools/device_frames_bench.py [--S 1,4,10] [--T 40] [--repeats 3] [--dry-run]"""
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


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='1,4,10', help='comma-separated sequence counts')
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--batch', type=int, default=10, help='frames per predict_batch call')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--gather-iters', type=int, default=200)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.S = sorted({int(s) for s in args.S.split(',')})
    except ValueError:
        ap.error('--S takes comma-separated integers')
    if min(args.S) < 1 or args.T < 2 or args.repeats < 1 or args.batch < 1 or args.gather_iters < 1:
        ap.error('need S >= 1, T >= 2, batch >= 1, repeats >= 1 and gather-iters >= 1')
    return args


def nv12_surface(img):
    """RGB uint8 [h,w,3] -> frames.NV12 over one [h*3/2, w] device surface (cv2's I420 with the chroma interleaved)."""
    import cv2
    import numpy as np
    import torch
    from gen6d_b200.frames import NV12
    h, w = img.shape[:2]
    i420 = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    surf = torch.from_numpy(np.vstack([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])).cuda()
    return NV12(surf[:h], surf[h:])


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'device_frames_bench', 'dry_run': True, 'S': args.S, 'T': args.T, 'batch': args.batch,
                          'repeats': args.repeats}))
        return
    import torch
    from gen6d_b200 import frames as fr, ops, synthetic as syn
    from golden import track_cases
    from instance_track_bench import video
    from track_bench import card

    T = args.T
    est, db = syn.build_estimator()
    idb = syn.synthetic_database(seed=7)
    iest = syn.build_estimator(idb)[0]
    K = db.K
    vids = [[db.render(p, K) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), T)] for s in range(max(args.S))]
    ivids = [video(idb, T, -8.0 * s) for s in range(max(args.S))]

    def replays(graphs):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for g in graphs:
            g.replay()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / 1e3

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def inputs(frames):
        """numpy frames per step -> {input: frames per step}, the device copies made once, before any timing."""
        return {'numpy': frames, 'rgb': [[torch.from_numpy(f).cuda() for f in step] for step in frames],
                'nv12': [[nv12_surface(f) for f in step] for step in frames]}

    def gather_time(step):
        """g6d_frames_gather alone over one step's device frames -> (microseconds per launch, MB moved)."""
        frames = fr.as_frames(step, 'bench', est.detector)
        plan = fr.FramePlan(fr.size_pattern(frames))
        table = plan.device_upload(est.detector, frames)[0]
        qn, (h, w) = len(frames), plan.pattern[0]
        # the launches captured in one graph, so the events time the kernels rather than the host's launch rate
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ops.frames_gather(table, qn, plan.H, plan.W, plan.nbytes)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.gather_iters):
                ops.frames_gather(table, qn, plan.H, plan.W, plan.nbytes)
        graph.replay()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        graph.replay()
        stop.record()
        torch.cuda.synchronize()
        read = sum(h * w * (1.5 if isinstance(f, fr.NV12) else 3) for f in frames)
        return round(start.elapsed_time(stop) / args.gather_iters * 1e3, 2), round((read + qn * h * w * 3) / 1e6, 2)

    def measure(label, S, per_frame, run, dev_graphs, ins):
        """run(frames per step) -> None (T steps end to end); dev_graphs: the numpy path's graphs of that schedule."""
        for k in ins:                                             # capture every input's graphs
            run(ins[k])
        runs = {k: [] for k in ('dev', 'numpy', 'rgb', 'nv12')}
        for _ in range(args.repeats):
            runs['dev'].append(per_frame / replays(dev_graphs()))
            for k in ('numpy', 'rgb', 'nv12'):
                runs[k].append(per_frame / timed(lambda: run(ins[k])))
        r = {k: round(statistics.median(v), 1) for k, v in runs.items()}
        g_rgb, g_nv12 = gather_time(ins['rgb'][0]), gather_time(ins['nv12'][0])
        r.update(what=label, S=S, runs={k: [round(x, 1) for x in v] for k, v in runs.items()},
                 gather_us={'rgb': g_rgb[0], 'nv12': g_nv12[0]}, gather_mb={'rgb': g_rgb[1], 'nv12': g_nv12[1]})
        print(json.dumps(r), file=sys.stderr, flush=True)
        return r

    res = []
    for S in args.S:
        frames = [[vids[s][t] for s in range(S)] for t in range(T)]
        ins = inputs(frames)
        trk = est.tracker(num_sequences=S)

        def run_trk(steps):
            trk.reset()
            for t in range(T):
                trk.step(steps[t], [K] * S)

        def trk_graphs():
            g = {k[0]: s.graph for k, s in trk.stages.stages.items() if isinstance(k[0], str)}
            return [g['track_full' if t == 0 else 'track_refine1'] for t in range(T)]
        res.append(measure('tracker', S, S * T, run_trk, trk_graphs, ins))
        trk.stages.clear()

        iframes = [[ivids[s][0][t] for s in range(S)] for t in range(T)]
        iKs = [ivids[s][1] for s in range(S)]
        ins = inputs(iframes)
        itrk = iest.instance_tracker(num_sequences=S, max_instances=2)

        def run_itrk(steps):
            itrk.reset()
            for t in range(T):
                itrk.step(steps[t], iKs)

        def itrk_graphs():
            g = {k[0]: s.graph for k, s in itrk.stages.stages.items() if isinstance(k[0], str)}
            return [g['detect' if t == 0 else 'refine'] for t in range(T)]
        res.append(measure('instance_tracker', S, S * T, run_itrk, itrk_graphs, ins))
        itrk.stages.clear()
        del ins
        torch.cuda.empty_cache()

    qn = args.batch
    batches = [[vids[(b + j) % len(vids)][(b * 3 + j) % T] for j in range(qn)] for b in range(4)]
    ins = inputs(batches)
    n_calls = max(4, T // 4)

    def run_pb(calls):
        for c in range(n_calls):
            est.predict_batch(calls[c % len(calls)], [K] * qn)

    def pb_graphs():
        return [next(s.graph for k, s in est.stages.stages.items() if k[0] == 'predict')] * n_calls
    res.append(measure('predict_batch', qn, qn * n_calls, run_pb, pb_graphs, ins))

    name, plimit = card()
    print(json.dumps({'tool': 'device_frames_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'repeats': args.repeats,
                      'refine_iter': est.cfg['refine_iter'], 'tracker_refine_iter': 1, 'frame_shape': [480, 640, 3],
                      'unit': 'sequence-frames/s (tracker, instance_tracker), frames/s (predict_batch)', 'results': res}))


if __name__ == '__main__':
    main()
