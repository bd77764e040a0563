"""Re-initialising single sequences of a lockstep tracker: S sequences x T rendered frames (the videos of
tools/track_bench.py) through Gen6DEstimator.tracker (device-glue path), one JSON line with the card and its power limit
read in the same run.  Every figure is the median of `--runs` alternating runs.
  * dev_ms: device-resident step time of the refine, mixed (m = 1 and m = S/2 re-initialised sequences) and full graphs
    (the captured graph replayed on frames already on the device);
  * e2e_fps: tracked frames/s end to end under three re-initialisation policies -- none, one sequence every 10 steps
    (round-robin), one sequence every step -- with reset(sequences) ('partial') and, for comparison, with reset() of all
    S sequences at the same steps ('full_reset');
  * objects: an ObjectTracker of K = 4 objects at the largest S under the every-10-steps policy;
  * max_memory_reserved_mb: torch.cuda.max_memory_reserved() once all of a tracker's graphs are captured.
  python tools/track_reinit_bench.py [--S 4,10] [--T 40] [--runs 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from gen6d_b200 import synthetic as syn  # noqa: E402
from track_bench import card  # noqa: E402
from golden import track_cases  # noqa: E402


def policy(name, S, t):
    """The sequences re-initialised before step t (t >= 1)."""
    if name == 'none':
        return []
    if name == 'every10':
        return [(t // 10) % S] if t % 10 == 0 else []
    return [t % S]                                                  # 'every_step'


def run_policy(trk, frames, Ks, name, partial):
    S = trk.S
    trk.reset()
    trk.step(frames[0], Ks)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(1, len(frames)):
        seqs = policy(name, S, t)
        if seqs:
            trk.reset(seqs) if partial else trk.reset()
        trk.step(frames[t], Ks)
    torch.cuda.synchronize()
    return S * (len(frames) - 1) / (time.perf_counter() - t0)


def replay_ms(stage, n=20):
    for _ in range(3):
        stage.graph.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        stage.graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='4,10')
    ap.add_argument('--T', type=int, default=40)
    ap.add_argument('--runs', type=int, default=3)
    args = ap.parse_args()
    est, db = syn.build_estimator()
    est.cfg['device_glue'] = True
    K = db.K
    med = lambda xs: round(float(np.median(xs)), 3)
    res = {}
    for S in [int(s) for s in args.S.split(',')]:
        videos = [[db.render(p, K) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), args.T)] for s in range(S)]
        frames = [[videos[s][t] for s in range(S)] for t in range(args.T)]
        Ks = [K] * S
        trk = None
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        trk = est.tracker(num_sequences=S)
        trk.step(frames[0], Ks)
        trk.step(frames[1], Ks)
        for m in range(1, S):                                       # capture every bucket's mixed graph
            trk.reset(list(range(m)))
            trk.step(frames[2], Ks)
        torch.cuda.synchronize()
        mem = torch.cuda.max_memory_reserved() / 2 ** 20
        stages = trk.stages.stages
        pick = lambda name: [s for k, s in stages.items() if k[0] == name][0]
        graphs = {'refine': pick('track_refine1'), 'full': pick('track_full'),
                  'mixed_m1': pick('track_mixed1'), f'mixed_m{S // 2}': pick(f'track_mixed{1 << (S // 2 - 1).bit_length()}')}
        dev = {k: [] for k in graphs}
        e2e = {f'{p}_{mode}': [] for p in ('none', 'every10', 'every_step') for mode in ('partial', 'full_reset')}
        for _ in range(args.runs):
            for k, st in graphs.items():
                dev[k].append(replay_ms(st))
            for p in ('none', 'every10', 'every_step'):
                for mode in ('partial', 'full_reset'):
                    e2e[f'{p}_{mode}'].append(run_policy(trk, frames, Ks, p, mode == 'partial'))
        res[S] = {'dev_ms': {k: med(v) for k, v in dev.items()}, 'e2e_fps': {k: med(v) for k, v in e2e.items()},
                  'mixed_graphs': len([k for k in stages if k[0].startswith('track_mixed')]),
                  'max_memory_reserved_mb': round(mem, 1)}
        print(json.dumps({'S': S, **res[S]}), file=sys.stderr, flush=True)
    # K = 4 objects at the largest S, one sequence every 10 steps
    del trk, graphs, stages
    torch.cuda.empty_cache()
    S = max(int(s) for s in args.S.split(','))
    objs = est.object_set()
    for i, seed in enumerate((7, 8, 11, 12)):
        objs.add(f'o{i}', syn.synthetic_database(seed=seed))
    otrk = objs.tracker(num_sequences=S)
    fps = {'partial': [], 'full_reset': []}
    for _ in range(args.runs):
        for mode in fps:
            fps[mode].append(run_policy(otrk, frames, Ks, 'every10', mode == 'partial') * len(objs))
    res['objects_K4'] = {'S': S, 'e2e_object_fps_every10': {k: med(v) for k, v in fps.items()}}
    name, plimit = card()
    print(json.dumps({'tool': 'track_reinit_bench', 'gpu': name, 'power_limit_w': plimit, 'T': args.T, 'runs': args.runs,
                      'results': res}))


if __name__ == '__main__':
    main()
