"""Re-detection schedules of the instance trackers (row f18): est.instance_tracker() on instance_track_bench.py's video
(two translating copies of the synthetic object at 480x640, T frames), cfg['refine_iter'] = 3, refine_iter = 1, M = 2.
One JSON line with the card and its power limit read in the same run; every rate and latency the median of --repeats
runs, the variants alternating.
  (a) S sequences stepped in lockstep, redetect_every = E, schedule 'lockstep' against 'staggered':
      instance-frames/s end to end (host clock around the T steps) and device-resident (CUDA events around each step's
      graph replay, summed); per-step latency median / p95 / max from the host clock around step() (it ends in its
      synchronising read) and from the CUDA events around the replay; graphs and kernels per graph; peak reserved MiB.
  (b) S streams under partial_track_bench.py's 'rates' (30/15/10 fps) and 'drops' schedules: one 'per_sequence' tracker
      stepped with sequences= against one num_sequences=1 tracker per stream: stream-frames/s, graphs, graph memory.
  python tools/instance_schedule_bench.py [--S 4,10] [--E 10] [--T 40] [--repeats 3] [--dry-run]"""
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

M = 2


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='4,10', help='comma-separated sequence counts')
    ap.add_argument('--E', type=int, default=10, help='redetect_every')
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.S = sorted({int(s) for s in args.S.split(',')})
    except ValueError:
        ap.error('--S takes comma-separated integers')
    if min(args.S) < 1 or args.E < 1 or args.T < 2 or args.repeats < 1:
        ap.error('need S >= 1, E >= 1, T >= 2 and repeats >= 1')
    return args


def pct(xs, q):
    import numpy as np
    return float(np.percentile(np.asarray(xs), q))


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'instance_schedule_bench', 'dry_run': True, 'S': args.S, 'E': args.E, 'T': args.T,
                          'repeats': args.repeats}))
        return
    import torch
    from gen6d_b200 import synthetic as syn
    from gen6d_b200.graphs import CapturedStage
    from instance_track_bench import video
    from partial_track_bench import schedule
    from track_bench import card

    db = syn.synthetic_database(seed=7)
    est = syn.build_estimator(db)[0]
    assert est.cfg['refine_iter'] == 3
    T = args.T
    seqs = [video(db, T, -8.0 * s) for s in range(max(args.S))]
    med = statistics.median

    # CUDA events around every graph replay of the run in progress
    events = []
    orig_call = CapturedStage.__call__

    def timed_call(self, *inputs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = orig_call(self, *inputs)
        b.record()
        events.append((a, b))
        return out
    CapturedStage.__call__ = timed_call

    def release(*trackers):
        for trk in trackers:
            trk.stages.clear()
        est.stages.clear()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        return torch.cuda.memory_reserved()

    res = {'lockstep_vs_staggered': [], 'rates_drops': [], 'skipped': []}
    for S in args.S:
        Ks = [seqs[s][1] for s in range(S)]
        row = {'S': S, 'M': M, 'E': args.E}
        try:
            base = release()
            trks = {sch: est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=args.E, schedule=sch)
                    for sch in ('lockstep', 'staggered')}
            stats = {sch: {'e2e': [], 'dev': [], 'host_ms': [], 'event_ms': []} for sch in trks}
            for rep in range(args.repeats + 1):                  # run 0 captures every graph (warm-up, not reported)
                for sch, trk in trks.items():
                    trk.reset()
                    host, ev = [], []
                    torch.cuda.synchronize()
                    t_all = time.perf_counter()
                    for t in range(T):
                        events.clear()
                        t0 = time.perf_counter()
                        trk.step([seqs[s][0][t] for s in range(S)], Ks)
                        host.append((time.perf_counter() - t0) * 1e3)
                        ev.append(sum(a.elapsed_time(b) for a, b in events))
                    wall = time.perf_counter() - t_all
                    if rep:
                        st = stats[sch]
                        st['e2e'].append(T * S * M / wall)
                        st['dev'].append(T * S * M / (sum(ev) / 1e3))
                        st['host_ms'].append(host)
                        st['event_ms'].append(ev)
            for sch, trk in trks.items():
                st = stats[sch]
                lat = lambda runs: {'median': med([med(r) for r in runs]), 'p95': med([pct(r, 95) for r in runs]),
                                    'max': med([max(r) for r in runs])}
                row[sch] = {'e2e_instance_fps': med(st['e2e']), 'dev_instance_fps': med(st['dev']),
                            'step_ms_host': lat(st['host_ms']), 'step_ms_events': lat(st['event_ms']),
                            'graphs': len(trk.stages.stages), 'kernels_per_graph': sorted(g.kernels for g in trk.stages.stages.values())}
            row['peak_reserved_mib'] = (torch.cuda.max_memory_reserved() - base) / 2 ** 20
            res['lockstep_vs_staggered'].append(row)
            del trks
        except torch.cuda.OutOfMemoryError:
            res['skipped'].append({'part': 'a', 'S': S, 'reason': 'out of memory'})
        # (b) streams at different rates: one per_sequence tracker against one tracker per stream
        for name in ('rates', 'drops'):
            sched = schedule(name, S, T)
            out = {'S': S, 'schedule': name}
            try:
                base = release()
                one = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=args.E, schedule='per_sequence')
                singles = [est.instance_tracker(num_sequences=1, max_instances=M, redetect_every=args.E) for _ in range(S)]
                fps = {'shared': [], 'per_stream': []}
                for rep in range(args.repeats + 1):
                    for kind in fps:
                        for trk in ([one] if kind == 'shared' else singles):
                            trk.reset()
                        torch.cuda.synchronize()
                        t0, n = time.perf_counter(), 0
                        for t, act in enumerate(sched):
                            if not act:
                                continue
                            if kind == 'shared':
                                one.step([seqs[s][0][t] for s in act], [Ks[s] for s in act], sequences=act)
                            else:
                                for s in act:
                                    singles[s].step([seqs[s][0][t]], [Ks[s]])
                            n += len(act)
                        torch.cuda.synchronize()
                        if rep:
                            fps[kind].append(n / (time.perf_counter() - t0))
                out.update({'stream_fps': {k: med(v) for k, v in fps.items()}, 'graphs_shared': len(one.stages.stages),
                            'graphs_per_stream': sum(len(s.stages.stages) for s in singles),
                            'peak_reserved_mib': (torch.cuda.max_memory_reserved() - base) / 2 ** 20})
                res['rates_drops'].append(out)
                del one, singles
            except torch.cuda.OutOfMemoryError:
                res['skipped'].append({'part': 'b', 'S': S, 'schedule': name, 'reason': 'out of memory'})
    CapturedStage.__call__ = orig_call
    release()
    name, plimit = card()
    print(json.dumps({'tool': 'instance_schedule_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'M': M,
                      'refine_iter_cfg': 3, 'refine_iter': 1, 'repeats': args.repeats, **res}))


if __name__ == '__main__':
    main()
