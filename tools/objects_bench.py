"""Several objects per frame: ObjectSet.predict (one shared query pyramid, one graph per call) against K single-object
estimators (K copies of the networks) running predict_batch back to back on the same frames.  One JSON line with the
card and its power limit read in the same run.  For each K (synthetic objects of seeds 7, 8, ...):
  * set_dev / est_dev: object-poses/s device-resident (the captured graphs replayed on frames already on the device);
  * set_e2e / est_e2e: object-poses/s end to end (numpy frames in, numpy poses out);
each the median of --repeats runs, the two variants alternating; peak_reserved_gb: the process's peak device memory.
  python tools/objects_bench.py [--K 1,2,4,8] [--frames 10] [--steps 10] [--repeats 3] [--dry-run]"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', default='1,2,4,8', help='comma-separated object counts')
    ap.add_argument('--frames', type=int, default=10, help='frames per batch (480x640)')
    ap.add_argument('--steps', type=int, default=10, help='timed calls per measurement')
    ap.add_argument('--repeats', type=int, default=3, help='alternating runs of the two variants; the median is reported')
    ap.add_argument('--refine-iter', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.K = sorted({int(k) for k in args.K.split(',') if k.strip()})
    except ValueError:
        ap.error(f'--K must be comma-separated integers, got {args.K!r}')
    if not args.K or min(args.K) < 1:
        ap.error('--K needs at least one object count, each >= 1')
    for name in ('frames', 'steps', 'repeats', 'refine_iter'):
        if getattr(args, name) < 1:
            ap.error(f'--{name.replace("_", "-")} must be >= 1')
    return args


def plan(args):
    """Databases, frames and calls of the run: frame i of a batch is view i of object i % K's database."""
    return {'seeds': [7 + k for k in range(max(args.K))], 'frame_shape': [480, 640, 3],
            'per_K': {K: {'frame_sources': [[7 + i % K, i] for i in range(args.frames)],
                          'object_poses_per_call': K * args.frames} for K in args.K},
            'steps': args.steps, 'repeats': args.repeats, 'refine_iter': args.refine_iter}


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'objects_bench', 'dry_run': True, 'plan': plan(args)}))
        return
    import numpy as np
    import torch
    from gen6d_b200 import synthetic as syn
    from track_bench import card

    seeds = plan(args)['seeds']
    dbs = [syn.synthetic_database(seed=s) for s in seeds]
    ests = [syn.build_estimator(db, refine_iter=args.refine_iter)[0] for db in dbs]   # one copy of the networks each
    objs = ests[0].object_set()                                                         # shares ests[0]'s networks
    res = {}

    def timed(fn, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def replayed(graphs, n):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(n):
            for g in graphs:
                g.replay()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / 1e3

    def release(stages):
        stages.clear()
        gc.collect()
        torch.cuda.empty_cache()

    for K in args.K:
        release(objs.stages)
        while len(objs) < K:
            objs.add(f'obj{len(objs)}', dbs[len(objs)])
        ids = [db.get_img_ids() for db in dbs[:K]]
        imgs = [np.asarray(dbs[i % K].get_image(ids[i % K][i])) for i in range(args.frames)]
        Ks = [dbs[i % K].get_K(ids[i % K][i]) for i in range(args.frames)]
        run_set = lambda: objs.predict(imgs, Ks)
        for _ in range(2):                                          # capture, then one warm call
            run_set()
        set_stage = next(iter(objs.stages.stages.values()))
        n = K * args.frames * args.steps
        runs = {'set_dev': [], 'est_dev': [], 'set_e2e': [], 'est_e2e': []}
        for _ in range(args.repeats):
            runs['set_dev'].append(n / replayed([set_stage.graph], args.steps))
            runs['set_e2e'].append(n / timed(run_set, args.steps))
            # the K estimators' graphs (one per estimator, several GB each at 10 frames) do not fit in 80 GB together
            # for K >= 4, so each estimator is captured, timed and released in turn; every predict_batch call ends in
            # a synchronising read, so back-to-back calls take the sum of these times
            t_dev = t_e2e = 0.0
            for e in ests[:K]:
                for _ in range(2):
                    e.predict_batch(imgs, Ks)
                graph = [s.graph for key, s in e.stages.stages.items() if key[0] == 'predict']
                assert len(graph) == 1
                t_dev += replayed(graph, args.steps)
                t_e2e += timed(lambda: e.predict_batch(imgs, Ks), args.steps)
                release(e.stages)
            runs['est_dev'].append(n / t_dev)
            runs['est_e2e'].append(n / t_e2e)
        res[K] = {k: round(statistics.median(v), 2) for k, v in runs.items()}
        res[K]['runs'] = {k: [round(x, 2) for x in v] for k, v in runs.items()}
        res[K].update(set_graph_kernels=set_stage.kernels, peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1))
        print(json.dumps({'K': K, **res[K]}), file=sys.stderr, flush=True)
        del set_stage
    name, plimit = card()
    print(json.dumps({'tool': 'objects_bench', 'gpu': name, 'power_limit_w': plimit, 'frames': args.frames,
                      'steps': args.steps, 'repeats': args.repeats, 'refine_iter': args.refine_iter,
                      'unit': 'object-poses/s', 'results': res}))


if __name__ == '__main__':
    main()
