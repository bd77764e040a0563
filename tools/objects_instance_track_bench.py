"""Multi-instance tracking of an object set: ObjectSet.instance_tracker() on synthetic videos of T frames (480x640) with
two copies of object a (seed 7), two of object b (seed 8) and one each of the further objects (seeds 11, 12) for K = 4,
composited without overlap (gen6d_b200.synthetic.instance_video), against K single-object est.instance_tracker()s (K
copies of the networks; each is captured, timed and released in turn, so their graphs never have to fit in memory
together, and their times are summed) and, at M = 1, against objs.tracker().  One JSON line with the card and its power
limit read in the same run.  For each (K, M, S, redetect_every) with K*M*S <= --max-crops:
  * set_dev / set_e2e: object-instance-frames/s (M slots x K objects x S sequences per step, live or not) over the
    T-step schedule, device-resident (the step graphs replayed on frames already on the device: detect on the
    re-detection steps, refine otherwise) and end to end (numpy frames in, numpy poses out);
  * singles_dev / singles_e2e: the same for the K single-object instance trackers back to back;
  * tracker_dev / tracker_e2e (M = 1 only): objs.tracker()'s object-frames/s over the same T steps;
  * graph_kernels: kernels in the set's detect and refine graphs, singles_graph_kernels the single trackers' summed;
    peak_reserved_gb: torch.cuda.max_memory_reserved() over the configuration (peak statistics reset before);
each rate the median of --repeats runs, the variants alternating.  Configurations over --max-crops are listed as skipped.
  python tools/objects_instance_track_bench.py [--K 1,2,4] [--M 1,2,4] [--S 1,4] [--redetect none,10] [--T 40]
                                               [--repeats 3] [--max-crops 40] [--dry-run]"""
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

SEEDS = (7, 8, 11, 12)
COPIES = (2, 2, 1, 1)             # copies of each object in the video


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', default='1,2,4', help='comma-separated object counts (at most 4)')
    ap.add_argument('--M', default='1,2,4', help='comma-separated max_instances')
    ap.add_argument('--S', default='1,4', help='comma-separated sequence counts')
    ap.add_argument('--redetect', default='none,10', help="comma-separated redetect_every values ('none': never)")
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--max-crops', type=int, default=40, help='skip configurations with K*M*S above this')
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.K = sorted({int(k) for k in args.K.split(',')})
        args.M = sorted({int(m) for m in args.M.split(',')})
        args.S = sorted({int(s) for s in args.S.split(',')})
        args.redetect = [None if v.strip().lower() == 'none' else int(v) for v in args.redetect.split(',')]
    except ValueError:
        ap.error('--K, --M, --S and --redetect take comma-separated integers (--redetect also "none")')
    if (min(args.K) < 1 or max(args.K) > len(SEEDS) or min(args.M) < 1 or max(args.M) > 16 or min(args.S) < 1
            or any(v is not None and v < 1 for v in args.redetect)):
        ap.error(f'need 1 <= K <= {len(SEEDS)}, 1 <= M <= 16, S >= 1 and redetect_every >= 1')
    if args.T < 2 or args.repeats < 1 or args.max_crops < 1:
        ap.error('need --T >= 2, --repeats >= 1 and --max-crops >= 1')
    return args


def plan(args):
    """-> (configurations to run, configurations skipped), each a (K, M, S, redetect_every) tuple."""
    run, skipped = [], []
    for K in args.K:
        for M in args.M:
            for S in args.S:
                for every in args.redetect:
                    (run if K * M * S <= args.max_crops else skipped).append((K, M, S, every))
    return run, skipped


def main():
    args = parse()
    run, skipped = plan(args)
    if args.dry_run:
        print(json.dumps({'tool': 'objects_instance_track_bench', 'dry_run': True, 'seeds': list(SEEDS[:max(args.K)]),
                          'copies': list(COPIES[:max(args.K)]), 'T': args.T, 'repeats': args.repeats, 'run': run,
                          'skipped': skipped}))
        print(f'dry run: {len(run)} configurations, {len(skipped)} skipped (K*M*S > {args.max_crops})')
        return
    import torch
    from gen6d_b200 import synthetic as syn
    from track_bench import card

    T, Kmax = args.T, max(args.K)
    dbs = [syn.synthetic_database(seed=s) for s in SEEDS[:Kmax]]
    ests = [syn.build_estimator(db)[0] for db in dbs]                 # one copy of the networks each
    objs = ests[0].object_set()                                         # shares ests[0]'s networks
    names = [f'obj{k}' for k in range(Kmax)]
    videos = {}

    def video(K, S):
        if (K, S) not in videos:
            seqs = [syn.instance_video(list(zip(dbs[:K], COPIES[:K])), T, -3.0 * s) for s in range(S)]
            videos[(K, S)] = ([[seqs[s][0][t] for s in range(S)] for t in range(T)], [seqs[s][1] for s in range(S)])
        return videos[(K, S)]

    def release(*trackers):
        for trk in trackers:
            trk.stages.clear()
        gc.collect()
        torch.cuda.empty_cache()

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

    def steps(trk, frames, Ks, n=T):
        trk.reset()
        for t in range(n):
            trk.step(frames[t], Ks)

    def itrack_schedule(trk, every):
        g = {k[0]: s for k, s in trk.stages.stages.items()}
        return [g['detect' if t == 0 or (every is not None and t % every == 0) else 'refine'].graph for t in range(T)], g

    res = []
    for K, M, S, every in run:
        frames, Ks = video(K, S)
        while len(objs) < K:
            objs.add(names[len(objs)], dbs[len(objs)])
        while len(objs) > K:
            objs.remove(names[len(objs) - 1])
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        kw = dict(num_sequences=S, max_instances=M, redetect_every=every)
        itrk = objs.instance_tracker(**kw)
        steps(itrk, frames, Ks)                                         # capture the graphs
        sched, sg = itrack_schedule(itrk, every)
        trk = objs.tracker(num_sequences=S) if M == 1 else None
        if trk is not None:
            steps(trk, frames, Ks, 2)
            tg = {k[0]: s for k, s in trk.stages.stages.items()}
            t_sched = [tg['track_full' if t == 0 else 'track_refine1'].graph for t in range(T)]
        n = M * K * S * T
        runs = {k: [] for k in ('set_dev', 'set_e2e', 'singles_dev', 'singles_e2e') + (('tracker_dev', 'tracker_e2e') if trk else ())}
        single_kernels = {'detect': 0, 'refine': 0}
        for rep in range(args.repeats):
            runs['set_dev'].append(n / replays(sched))
            runs['set_e2e'].append(n / timed(lambda: steps(itrk, frames, Ks)))
            if trk is not None:
                runs['tracker_dev'].append(K * S * T / replays(t_sched))
                runs['tracker_e2e'].append(K * S * T / timed(lambda: steps(trk, frames, Ks)))
            t_dev = t_e2e = 0.0
            for e in ests[:K]:                                          # each single tracker captured, timed, released
                one = e.instance_tracker(**kw)
                steps(one, frames, Ks)
                o_sched, og = itrack_schedule(one, every)
                if rep == 0:
                    for k in single_kernels:
                        single_kernels[k] += og[k].kernels
                t_dev += replays(o_sched)
                t_e2e += timed(lambda: steps(one, frames, Ks))
                del o_sched, og
                release(one)
            runs['singles_dev'].append(n / t_dev)
            runs['singles_e2e'].append(n / t_e2e)
        r = {k: round(statistics.median(v), 1) for k, v in runs.items()}
        r.update(K=K, M=M, S=S, redetect_every=every, runs={k: [round(x, 1) for x in v] for k, v in runs.items()},
                 graph_kernels={'detect': sg['detect'].kernels, 'refine': sg['refine'].kernels},
                 singles_graph_kernels=single_kernels, peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1))
        res.append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
        del sched, sg
        if trk is not None:
            del tg, t_sched
            release(trk)
        release(itrk)
    name, plimit = card()
    print(json.dumps({'tool': 'objects_instance_track_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T,
                      'repeats': args.repeats, 'refine_iter': ests[0].cfg['refine_iter'], 'frame_shape': [480, 640, 3],
                      'unit': 'object-instance-frames/s (set_*, singles_*), object-frames/s (tracker_*)',
                      'skipped': [dict(K=K, M=M, S=S, redetect_every=e) for K, M, S, e in skipped], 'results': res}))


if __name__ == '__main__':
    main()
