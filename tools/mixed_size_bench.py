"""Frames of different sizes (DESIGN.md row f13): ONE lockstep tracker over S sequences spread over two or three frame
sizes against one tracker per size stepped back to back (what a user without mixed-size support runs).  The sequences are
crops of a synthetic video of T frames in which two copies of the object translate (tools/instance_track_bench.py's
video): 480x640 itself, 448x576 and 384x512, principal points shifted to match.  One JSON line with the card and its
power limit read in the same run.  For each (S, number of sizes):
  * tracker / itrack / itrack_re10: est.tracker(), est.instance_tracker() (max_instances 2) and the same with
    redetect_every=10, tracker refine_iter 1, cfg refine_iter 3; '<kind>_mixed_dev' / '<kind>_per_size_dev': frames/s
    (sequence-frames, one per sequence and step) over the T-step schedule replaying the step graphs on frames already on
    the device, '_e2e' the same end to end (numpy frames in, numpy poses out);
  * predict_batch_mixed / predict_batch_per_size: frames/s of predict_batch on the S frames of step 0 as one mixed batch
    against one batch per size, device-resident and end to end;
  * graph_kernels: kernels per graph; peak_reserved_gb: torch.cuda.max_memory_reserved() per kind (statistics reset
    before, every other graph released);
each rate the median of --repeats runs, the two variants alternating.
  python tools/mixed_size_bench.py [--S 4,10] [--sizes 2,3] [--T 40] [--repeats 3] [--dry-run]"""
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

CROPS = [(0, 0, 480, 640), (16, 32, 448, 576), (48, 64, 384, 512)]       # (y0, x0, h, w) of the 480x640 frames


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='4,10', help='comma-separated sequence counts')
    ap.add_argument('--sizes', default='2,3', help='comma-separated numbers of frame sizes (2 or 3)')
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.S = sorted({int(s) for s in args.S.split(',')})
        args.sizes = sorted({int(s) for s in args.sizes.split(',')})
    except ValueError:
        ap.error('--S and --sizes take comma-separated integers')
    if min(args.sizes) < 2 or max(args.sizes) > len(CROPS) or any(s < z for s in args.S for z in args.sizes):
        ap.error(f'need 2 <= sizes <= {len(CROPS)} and S >= sizes')
    if args.T < 2 or args.repeats < 1:
        ap.error('need --T >= 2 and --repeats >= 1')
    return args


def crop(img, K, z):
    import numpy as np
    y0, x0, h, w = CROPS[z]
    K = np.array(K, np.float64)
    K[0, 2] -= x0
    K[1, 2] -= y0
    return np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w]), K


def kind_of(key):
    """A StageCache key's graph kind: the plain name, or the name inside a size pattern's key."""
    name = key[0]
    while isinstance(name, tuple):
        name = name[0]
    return name


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'mixed_size_bench', 'dry_run': True, 'S': args.S, 'sizes': args.sizes, 'T': args.T,
                          'repeats': args.repeats, 'crops': CROPS}))
        return
    import torch
    from gen6d_b200 import synthetic as syn
    from instance_track_bench import video
    from track_bench import card

    db = syn.synthetic_database(seed=7)
    est = syn.build_estimator(db)[0]                # cfg refine_iter 3
    T = args.T
    seqs = [video(db, T, -8.0 * s) for s in range(max(args.S))]

    def release(*holders):
        for h in holders:
            h.stages.clear()
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

    makers = {'tracker': lambda n: est.tracker(num_sequences=n),
              'itrack': lambda n: est.instance_tracker(num_sequences=n, max_instances=2),
              'itrack_re10': lambda n: est.instance_tracker(num_sequences=n, max_instances=2, redetect_every=10)}
    res = []
    for S in args.S:
        for nz in args.sizes:
            zs = [s % nz for s in range(S)]
            frames, Ks = [], None
            for t in range(T):
                out = [crop(seqs[s][0][t], seqs[s][1], zs[s]) for s in range(S)]
                frames.append([o[0] for o in out])
                Ks = [o[1] for o in out]
            groups = [[s for s in range(S) if zs[s] == z] for z in range(nz)]
            r = {'S': S, 'sizes': [list(CROPS[z][2:]) for z in range(nz)], 'sequences_per_size': [len(g) for g in groups],
                 'graph_kernels': {}, 'peak_reserved_gb': {}, 'runs': {}}
            for kind, make in makers.items():
                release()
                torch.cuda.reset_peak_memory_stats()
                mixed, per = make(S), [make(len(g)) for g in groups]

                def run_mixed():
                    mixed.reset()
                    for t in range(T):
                        mixed.step(frames[t], Ks)

                def run_per():
                    for trk in per:
                        trk.reset()
                    for t in range(T):
                        for trk, g in zip(per, groups):
                            trk.step([frames[t][i] for i in g], [Ks[i] for i in g])

                run_mixed()                                      # capture the graphs
                run_per()
                first = {'tracker': 'track_full', 'itrack': 'detect', 'itrack_re10': 'detect'}[kind]
                later = {'tracker': 'track_refine1', 'itrack': 'refine', 'itrack_re10': 'refine'}[kind]
                every = 10 if kind == 'itrack_re10' else None
                sched = [first if t == 0 or (every and t % every == 0) else later for t in range(T)]
                graphs = lambda trk: {kind_of(k): s for k, s in trk.stages.stages.items()}
                gm, gp = graphs(mixed), [graphs(trk) for trk in per]
                m_sched = [gm[n].graph for n in sched]
                p_sched = [g[n].graph for n in sched for g in gp]
                runs = {f'{kind}_mixed_dev': [], f'{kind}_per_size_dev': [], f'{kind}_mixed_e2e': [], f'{kind}_per_size_e2e': []}
                for _ in range(args.repeats):
                    runs[f'{kind}_mixed_dev'].append(S * T / replays(m_sched))
                    runs[f'{kind}_per_size_dev'].append(S * T / replays(p_sched))
                    runs[f'{kind}_mixed_e2e'].append(S * T / timed(run_mixed))
                    runs[f'{kind}_per_size_e2e'].append(S * T / timed(run_per))
                for k, v in runs.items():
                    r[k] = round(statistics.median(v), 1)
                    r['runs'][k] = [round(x, 1) for x in v]
                r['graph_kernels'][kind] = {'mixed': {n: s.kernels for n, s in gm.items()},
                                            'per_size': [{n: s.kernels for n, s in g.items()} for g in gp]}
                r['peak_reserved_gb'][kind] = round(torch.cuda.max_memory_reserved() / 2 ** 30, 2)
                del gm, gp, m_sched, p_sched
                release(mixed, *per)
            # predict_batch on the S frames of step 0: one mixed batch against one batch per size
            release()
            torch.cuda.reset_peak_memory_stats()
            f0 = frames[0]
            pb_mixed = lambda: est.predict_batch(f0, Ks)
            pb_per = lambda: [est.predict_batch([f0[i] for i in g], [Ks[i] for i in g]) for g in groups]
            pb_mixed()
            pb_per()
            mixed_g = [s.graph for k, s in est.stages.stages.items() if isinstance(k[0], tuple)]
            per_g = [s.graph for k, s in est.stages.stages.items() if not isinstance(k[0], tuple)]
            runs = {'predict_batch_mixed_dev': [], 'predict_batch_per_size_dev': [], 'predict_batch_mixed_e2e': [],
                    'predict_batch_per_size_e2e': []}
            reps = 10
            for _ in range(args.repeats):
                runs['predict_batch_mixed_dev'].append(S * reps / replays(mixed_g * reps))
                runs['predict_batch_per_size_dev'].append(S * reps / replays(per_g * reps))
                runs['predict_batch_mixed_e2e'].append(S * reps / timed(lambda: [pb_mixed() for _ in range(reps)]))
                runs['predict_batch_per_size_e2e'].append(S * reps / timed(lambda: [pb_per() for _ in range(reps)]))
            for k, v in runs.items():
                r[k] = round(statistics.median(v), 1)
                r['runs'][k] = [round(x, 1) for x in v]
            r['graph_kernels']['predict_batch'] = {'mixed': [s.kernels for k, s in est.stages.stages.items() if isinstance(k[0], tuple)],
                                                   'per_size': [s.kernels for k, s in est.stages.stages.items()
                                                                if not isinstance(k[0], tuple)]}
            r['peak_reserved_gb']['predict_batch'] = round(torch.cuda.max_memory_reserved() / 2 ** 30, 2)
            del mixed_g, per_g
            release()
            res.append(r)
            print(json.dumps(r), file=sys.stderr, flush=True)
    name, plimit = card()
    print(json.dumps({'tool': 'mixed_size_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'repeats': args.repeats,
                      'refine_iter': est.cfg['refine_iter'], 'tracker_refine_iter': 1, 'max_instances': 2,
                      'unit': 'sequence-frames/s', 'results': res}))


if __name__ == '__main__':
    main()
