"""Device frames at a working resolution (row f15): what resizing decoder surfaces inside the graph buys, on T frames
rendered at 540x960 and upscaled once, before any timing, to 1080x1920 NV12 surfaces on the device (cfg['refine_iter'] =
3, tracker refine_iter = 1).  One JSON line with the card and its power limit read in the same run.

(a) gather: g6d_frames_gather_resized alone, 1 and 10 random NV12 frames at 1080x1920 and 2160x3840 to 960 on the long
    side (CUDA events over --gather-iters launches captured in one graph, the median of --repeats runs).  mb: the NV12
    source surfaces plus the RGB working images written, computed from shapes.
(b) est.tracker() and est.instance_tracker(max_instances=2) at each S, and predict_batch on --batch frames, fed three
    ways, timed alternately, each the median of --repeats runs:
      * resized: Resized(nv12, max_side=960), the working 540x960 frames gathered in the graph;
      * host:    the workaround without it: each surface downloaded, cv2.cvtColor(COLOR_YUV2RGB_NV12) and cv2.resize to
                 960x540 on the host, the numpy path;
      * full:    the 1080x1920 surface as it is (detection and crops at full size, K scaled to it).
    e2e: sequence-frames/s end to end (frames/s for predict_batch); dev: the same schedule's captured graphs replayed
    alone (device-resident, no input preparation, no read); graph_kernels: kernels per captured graph;
    peak_reserved_gb: torch.cuda.max_memory_reserved() over a capturing run of that feed alone (no other feed's graphs
    alive, cache emptied, statistics reset before).
  python tools/resized_frames_bench.py [--S 1,4,10] [--T 40] [--repeats 3] [--dry-run]"""
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

FEEDS = ('resized', 'host', 'full')


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


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'resized_frames_bench', 'dry_run': True, 'S': args.S, 'T': args.T, 'batch': args.batch,
                          'repeats': args.repeats, 'feeds': FEEDS}))
        return
    import cv2
    import numpy as np
    import torch
    from device_frames_bench import nv12_surface
    from gen6d_b200 import frames as fr, ops, synthetic as syn
    from golden import track_cases
    from track_bench import card

    T, med = args.T, statistics.median
    db = syn.synthetic_database(height=540, width=960)
    est = syn.build_estimator(db)[0]
    K = db.K.astype(np.float64)
    K_full = np.array([[2.0, 0, 0.5], [0, 2.0, 0.5], [0, 0, 1]]) @ K       # the same camera on the 2x source
    up = lambda img: cv2.resize(img, (1920, 1080), interpolation=cv2.INTER_LINEAR)
    vids = [[nv12_surface(up(db.render(p, db.K))) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), T)]
            for s in range(max(args.S))]
    torch.cuda.synchronize()

    def event_time(fn):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / 1e3

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    # ---------------------------------------------------------------- (a) the gather alone
    gather = []
    for (h, w) in ((1080, 1920), (2160, 3840)):
        for n in (1, 10):
            g = torch.Generator(device='cuda').manual_seed(n)
            surf = [torch.randint(0, 256, (h * 3 // 2, w), dtype=torch.uint8, device='cuda', generator=g) for _ in range(n)]
            frames = fr.as_frames([fr.Resized(fr.NV12(s[:h], s[h:]), max_side=960) for s in surf], 'bench', est.detector)
            plan = fr.FramePlan(fr.size_pattern(frames))
            table = plan.device_upload(est.detector, frames, True)[0]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                ops.frames_gather_resized(table, n, plan.H, plan.W, plan.nbytes)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(args.gather_iters):
                    ops.frames_gather_resized(table, n, plan.H, plan.W, plan.nbytes)
            graph.replay()
            runs = [event_time(graph.replay) / args.gather_iters * 1e6 for _ in range(args.repeats)]
            rh, rw = plan.pattern[0]
            mb = n * (h * w * 1.5 + rh * rw * 3) / 1e6
            gather.append({'src': [h, w], 'frames': n, 'working': [rh, rw], 'us': round(med(runs), 2),
                           'runs_us': [round(x, 2) for x in runs], 'mb': round(mb, 2), 'gb_s': round(mb / 1e3 / (med(runs) / 1e6), 1)})
            print(json.dumps(gather[-1]), file=sys.stderr, flush=True)
            del graph, surf, frames, table

    # ---------------------------------------------------------------- (b) whole steps, three feeds
    def host_rgb(f):
        yuv = np.vstack([f.y.cpu().numpy(), f.uv.cpu().numpy()])
        return cv2.resize(cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12), (960, 540), interpolation=cv2.INTER_LINEAR)

    feed = {'resized': (lambda fs: [fr.Resized(f, max_side=960) for f in fs], K),
            'host': (lambda fs: [host_rgb(f) for f in fs], K),
            'full': (lambda fs: list(fs), K_full)}

    def graph_of(stages, name):
        """The captured stage of graph `name` in any feed's key: 'name', ('device', 'name', ...), ('device-resized', ...)."""
        for k, s in stages.items():
            if k[0] == name or (isinstance(k[0], tuple) and len(k[0]) == 3 and k[0][1] == name):
                return s
        raise KeyError(name)

    def measure(label, S, per_frame, run, stages, schedule):
        """run(feed) -> None (the whole schedule end to end); stages() -> the StageCache's dict, cleared between feeds;
        schedule: the graph name of each step."""
        out = {'what': label, 'S': S, 'runs': {f: {'e2e': [], 'dev': []} for f in FEEDS}, 'graph_kernels': {}, 'peak_reserved_gb': {}}
        for f in FEEDS:                                   # each feed's memory alone: no other feed's graphs alive
            stages().clear()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            run(f)
            out['peak_reserved_gb'][f] = round(torch.cuda.max_memory_reserved() / 2 ** 30, 2)
            out['graph_kernels'][f] = {n: graph_of(stages(), n).kernels for n in dict.fromkeys(schedule)}
        graphs = {}
        for f in FEEDS:                                   # then every feed's graphs captured and kept for the alternation
            stages().clear()
            torch.cuda.empty_cache()
            run(f)
            graphs[f] = dict(stages())
        for _ in range(args.repeats):
            for f in FEEDS:
                stages().clear()
                stages().update(graphs[f])
                seq = [graph_of(graphs[f], n).graph for n in schedule]
                out['runs'][f]['dev'].append(per_frame / event_time(lambda: [g.replay() for g in seq]))
                out['runs'][f]['e2e'].append(per_frame / timed(lambda: run(f)))
        for f in FEEDS:
            out[f] = {k: round(med(v), 1) for k, v in out['runs'][f].items()}
            out['runs'][f] = {k: [round(x, 1) for x in v] for k, v in out['runs'][f].items()}
        stages().clear()
        print(json.dumps(out), file=sys.stderr, flush=True)
        return out

    res = []
    for S in args.S:
        steps = [[vids[s][t] for s in range(S)] for t in range(T)]
        trk = est.tracker(num_sequences=S)

        def run_trk(f):
            make, Kf = feed[f]
            trk.reset()
            for t in range(T):
                trk.step(make(steps[t]), [Kf] * S)
        res.append(measure('tracker', S, S * T, run_trk, lambda: trk.stages.stages,
                           ['track_full'] + ['track_refine1'] * (T - 1)))

        itrk = est.instance_tracker(num_sequences=S, max_instances=2)

        def run_itrk(f):
            make, Kf = feed[f]
            itrk.reset()
            for t in range(T):
                itrk.step(make(steps[t]), [Kf] * S)
        res.append(measure('instance_tracker', S, S * T, run_itrk, lambda: itrk.stages.stages, ['detect'] + ['refine'] * (T - 1)))
        del trk, itrk
        torch.cuda.empty_cache()

    qn = args.batch
    batches = [[vids[(b + j) % len(vids)][(b * 3 + j) % T] for j in range(qn)] for b in range(4)]
    n_calls = max(4, T // 4)

    def run_pb(f):
        make, Kf = feed[f]
        for c in range(n_calls):
            est.predict_batch(make(batches[c % len(batches)]), [Kf] * qn)
    res.append(measure('predict_batch', qn, qn * n_calls, run_pb, lambda: est.stages.stages, ['predict'] * n_calls))

    name, plimit = card()
    print(json.dumps({'tool': 'resized_frames_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'repeats': args.repeats,
                      'refine_iter': est.cfg['refine_iter'], 'tracker_refine_iter': 1, 'source_shape': [1080, 1920],
                      'working_shape': [540, 960],
                      'unit': 'sequence-frames/s (tracker, instance_tracker), frames/s (predict_batch)', 'gather': gather,
                      'results': res}))


if __name__ == '__main__':
    main()
