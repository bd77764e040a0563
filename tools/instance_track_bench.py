"""Multi-instance tracking: Gen6DEstimator.instance_tracker() on a synthetic video of T frames (480x640) in which two
copies of the synthetic object translate across the frame (composited as tests/test_instances_gpu.py does), against
est.tracker() (one instance per sequence) and predict_instances on every frame.  One JSON line with the card and its power
limit read in the same run.  For each (S, M, redetect_every):
  * itrack_dev / itrack_e2e: instance-frames/s (M slots x S sequences per step, live or not) over the T-step schedule,
    device-resident (the step graphs replayed on frames already on the device: detect on the re-detection steps, refine
    otherwise) and end to end (numpy frames in, numpy poses out);
  * tracker_dev / tracker_e2e: est.tracker()'s frames/s over the same T steps (one pose per sequence);
  * instances_dev / instances_e2e: predict_instances instance-frames/s with a call per step (a full prediction each);
  * graph_kernels: kernels in the detect and refine graphs; peak_reserved_gb: torch.cuda.max_memory_reserved() over the
    configuration (peak statistics reset before; every other graph released);
each rate the median of --repeats runs, the variants alternating.
  python tools/instance_track_bench.py [--S 1,4,10] [--M 1,2,4] [--redetect none,10] [--T 40] [--repeats 3] [--dry-run]"""
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
    ap.add_argument('--S', default='1,4,10', help='comma-separated sequence counts')
    ap.add_argument('--M', default='1,2,4', help='comma-separated max_instances')
    ap.add_argument('--redetect', default='none,10', help="comma-separated redetect_every values ('none': never)")
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.S = sorted({int(s) for s in args.S.split(',')})
        args.M = sorted({int(m) for m in args.M.split(',')})
        args.redetect = [None if v.strip().lower() == 'none' else int(v) for v in args.redetect.split(',')]
    except ValueError:
        ap.error('--S, --M and --redetect take comma-separated integers (--redetect also "none")')
    if min(args.S) < 1 or min(args.M) < 1 or max(args.M) > 16 or any(v is not None and v < 1 for v in args.redetect):
        ap.error('need S >= 1, 1 <= M <= 16 and redetect_every >= 1')
    if args.T < 2 or args.repeats < 1:
        ap.error('need --T >= 2 and --repeats >= 1')
    return args


def video(db, T, shift):
    """T frames of two copies of the object moving 4 px per frame to the right."""
    import numpy as np
    i = db.get_img_ids()[3]
    pose, K = db.poses[i].copy(), db.get_K(i)
    frames = []
    for t in range(T):
        dx = shift + 4.0 * t
        a, b = pose.copy(), pose.copy()
        a[0, 3] += (dx - 120.0) * pose[2, 3] / K[0, 0]
        b[0, 3] += (dx + 220.0) * pose[2, 3] / K[0, 0]
        ia, ib = db.render(a, K), db.render(b, K)
        frames.append(np.where((ib != db._bg).any(-1, keepdims=True), ib, ia))
    return frames, K


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'instance_track_bench', 'dry_run': True, 'S': args.S, 'M': args.M, 'redetect': args.redetect,
                          'T': args.T, 'repeats': args.repeats}))
        return
    import numpy as np
    import torch
    from gen6d_b200 import synthetic as syn
    from track_bench import card

    db = syn.synthetic_database(seed=7)
    est = syn.build_estimator(db)[0]
    T = args.T
    seqs = [video(db, T, -8.0 * s) for s in range(max(args.S))]

    def release(*trackers):
        for trk in trackers:
            trk.stages.clear()
        est.stages.clear()
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

    res = []
    for S in args.S:
        frames = [[seqs[s][0][t] for s in range(S)] for t in range(T)]
        Ks = [seqs[s][1] for s in range(S)]
        for M in args.M:
            for every in args.redetect:
                release()
                torch.cuda.reset_peak_memory_stats()
                itrk, trk = est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=every), est.tracker(num_sequences=S)
                detect_at = [t == 0 or (every is not None and t % every == 0) for t in range(T)]

                def run_itrk():
                    itrk.reset()
                    for t in range(T):
                        itrk.step(frames[t], Ks)

                def run_trk():
                    trk.reset()
                    for t in range(T):
                        trk.step(frames[t], Ks)

                def run_inst():
                    for t in range(T):
                        est.predict_instances(frames[t], Ks, max_instances=M)

                run_itrk()                                           # capture the graphs
                for t in range(2):
                    trk.step(frames[t], Ks)
                    est.predict_instances(frames[t], Ks, max_instances=M)
                ig = {k[0]: s for k, s in itrk.stages.stages.items()}
                tg = {k[0]: s for k, s in trk.stages.stages.items()}
                pg = next(s for k, s in est.stages.stages.items() if k[0][0] == 'instances')
                i_sched = [ig['detect' if d else 'refine'].graph for d in detect_at]
                t_sched = [tg['track_full' if t == 0 else 'track_refine1'].graph for t in range(T)]
                runs = {k: [] for k in ('itrack_dev', 'itrack_e2e', 'tracker_dev', 'tracker_e2e', 'instances_dev', 'instances_e2e')}
                for _ in range(args.repeats):
                    runs['itrack_dev'].append(M * S * T / replays(i_sched))
                    runs['tracker_dev'].append(S * T / replays(t_sched))
                    runs['instances_dev'].append(M * S * T / replays([pg.graph] * T))
                    runs['itrack_e2e'].append(M * S * T / timed(run_itrk))
                    runs['tracker_e2e'].append(S * T / timed(run_trk))
                    runs['instances_e2e'].append(M * S * T / timed(run_inst))
                r = {k: round(statistics.median(v), 1) for k, v in runs.items()}
                r.update(S=S, M=M, redetect_every=every, runs={k: [round(x, 1) for x in v] for k, v in runs.items()},
                         graph_kernels={'detect': ig['detect'].kernels, 'refine': ig['refine'].kernels},
                         tracker_graph_kernels={'full': tg['track_full'].kernels, 'refine': tg['track_refine1'].kernels},
                         instances_graph_kernels=pg.kernels,
                         peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1))
                res.append(r)
                print(json.dumps(r), file=sys.stderr, flush=True)
                del ig, tg, pg, i_sched, t_sched
                release(itrk, trk)
    name, plimit = card()
    print(json.dumps({'tool': 'instance_track_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'repeats': args.repeats,
                      'refine_iter': est.cfg['refine_iter'], 'frame_shape': [480, 640, 3],
                      'unit': 'instance-frames/s (itrack_*, instances_*), frames/s (tracker_*)', 'results': res}))


if __name__ == '__main__':
    main()
