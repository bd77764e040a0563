"""Several instances per frame: Gen6DEstimator.predict_instances (the detector once, M crops / selections / refinements
per frame, one graph per call) against predict_batch on the same frames.  One JSON line with the card and its power limit
read in the same run.  For each M:
  * inst_dev / inst_e2e: instance-poses/s (M poses per frame, valid or not) device-resident (the captured graph replayed on
    frames already on the device) and end to end (numpy frames in, numpy poses out);
  * batch_dev / batch_e2e: predict_batch poses/s on the same frames (one pose per frame), and inst_dev / batch_dev;
  * graph_kernels: kernels in predict_instances' graph (predict_batch's: batch_graph_kernels);
  * peak_reserved_gb: torch.cuda.max_memory_reserved() over that M's capture and timing (peak statistics reset before);
each rate the median of --repeats runs, the two variants alternating.
  python tools/instances_bench.py [--M 1,2,4,8] [--frames 10] [--steps 10] [--repeats 3] [--dry-run]"""
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
    ap.add_argument('--M', default='1,2,4,8', help='comma-separated instance counts (max_instances)')
    ap.add_argument('--frames', type=int, default=10, help='frames per batch (480x640)')
    ap.add_argument('--steps', type=int, default=10, help='timed calls per measurement')
    ap.add_argument('--repeats', type=int, default=3, help='alternating runs of the two variants; the median is reported')
    ap.add_argument('--refine-iter', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.M = sorted({int(m) for m in args.M.split(',') if m.strip()})
    except ValueError:
        ap.error(f'--M must be comma-separated integers, got {args.M!r}')
    if not args.M or min(args.M) < 1 or max(args.M) > 16:
        ap.error('--M needs at least one instance count, each in [1, 16]')
    for name in ('frames', 'steps', 'repeats', 'refine_iter'):
        if getattr(args, name) < 1:
            ap.error(f'--{name.replace("_", "-")} must be >= 1')
    return args


def plan(args):
    return {'seed': 7, 'frame_shape': [480, 640, 3], 'frames': args.frames,
            'per_M': {M: {'instance_poses_per_call': M * args.frames} for M in args.M},
            'steps': args.steps, 'repeats': args.repeats, 'refine_iter': args.refine_iter}


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'instances_bench', 'dry_run': True, 'plan': plan(args)}))
        return
    import numpy as np
    import torch
    from gen6d_b200 import synthetic as syn
    from track_bench import card

    db = syn.synthetic_database(seed=plan(args)['seed'])
    est = syn.build_estimator(db, refine_iter=args.refine_iter)[0]
    ids = db.get_img_ids()
    imgs = [np.asarray(db.get_image(ids[i % len(ids)])) for i in range(args.frames)]
    Ks = [db.get_K(ids[i % len(ids)]) for i in range(args.frames)]
    res = {}

    def timed(fn, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def replayed(graph, n):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(n):
            graph.replay()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / 1e3

    def release():
        est.stages.clear()
        gc.collect()
        torch.cuda.empty_cache()

    for M in args.M:
        release()
        torch.cuda.reset_peak_memory_stats()
        run_inst = lambda: est.predict_instances(imgs, Ks, max_instances=M)
        run_batch = lambda: est.predict_batch(imgs, Ks)
        for _ in range(2):                                          # capture, then one warm call
            run_inst()
            run_batch()
        stages = {key[0] if isinstance(key[0], str) else key[0][0]: s for key, s in est.stages.stages.items()}
        inst, batch = stages['instances'], stages['predict']
        n = args.frames * args.steps
        runs = {'inst_dev': [], 'batch_dev': [], 'inst_e2e': [], 'batch_e2e': []}
        for _ in range(args.repeats):
            runs['inst_dev'].append(M * n / replayed(inst.graph, args.steps))
            runs['batch_dev'].append(n / replayed(batch.graph, args.steps))
            runs['inst_e2e'].append(M * n / timed(run_inst, args.steps))
            runs['batch_e2e'].append(n / timed(run_batch, args.steps))
        r = {k: round(statistics.median(v), 2) for k, v in runs.items()}
        r['inst_over_batch_dev'] = round(r['inst_dev'] / r['batch_dev'], 3)
        r['runs'] = {k: [round(x, 2) for x in v] for k, v in runs.items()}
        _, inter = run_inst()
        r.update(graph_kernels=inst.kernels, batch_graph_kernels=batch.kernels,
                 mean_valid_instances=round(float(inter['instance_count'].mean()), 2),
                 peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1))
        res[M] = r
        print(json.dumps({'M': M, **r}), file=sys.stderr, flush=True)
        del inst, batch, stages
    name, plimit = card()
    print(json.dumps({'tool': 'instances_bench', 'gpu': name, 'power_limit_w': plimit, 'frames': args.frames,
                      'steps': args.steps, 'repeats': args.repeats, 'refine_iter': args.refine_iter,
                      'unit': 'instance-poses/s (inst_*), poses/s (batch_*)', 'results': res}))


if __name__ == '__main__':
    main()
