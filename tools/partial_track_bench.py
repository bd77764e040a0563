"""Streams at different frame rates through one tracker (row f17): S streams x T ticks of rendered 480x640 frames, each
stream active on a tick by a schedule, through one Gen6DEstimator.tracker stepped with sequences= (the active streams),
against one num_sequences=1 tracker per stream stepped back to back (the other correct option).  One JSON line with the
card and its power limit read in the same run; every figure is the median of `--runs` alternating runs.
  * schedules: 'rates' (stream s active when t % (1 + s % 3) == 0: 30/15/10 fps on a 30 Hz tick), 'drops' (each frame
    dropped with p = 0.2, seeded), 'all' (every stream every tick, the lockstep ceiling);
  * e2e_fps: tracked stream-frames/s end to end (numpy frames: upload, replays, reads);
  * dev_fps: tracked stream-frames/s device-resident (each tick's captured graphs replayed on frames already on the
    device);
  * graphs / kernels: graphs captured and kernel nodes per graph; graph_memory_mb: the peak memory torch reserves while
    an option's trackers capture all their graphs, above what was reserved before (its trackers' state and graph pools);
  * objects: an ObjectTracker of K = 2 objects at the largest S under 'rates' (tracked object-frames/s).
  python tools/partial_track_bench.py [--S 4,10] [--T 60] [--runs 3] [--refine-iter 1]"""
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


def schedule(name, S, T, seed=0):
    """The active streams of every tick (ascending); tick 0 has every stream (their first frames)."""
    rng = np.random.RandomState(seed)
    out = []
    for t in range(T):
        if name == 'rates':
            act = [s for s in range(S) if t % (1 + s % 3) == 0]
        elif name == 'drops':
            act = [s for s in range(S) if t == 0 or rng.rand() >= 0.2]
        else:
            act = list(range(S))
        out.append(act)
    return out


def run_partial(trk, frames, Ks, sched):
    """One tracker, sequences= the active streams -> stream-frames/s."""
    trk.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for t, act in enumerate(sched):
        if act:
            trk.step([frames[t][s] for s in act], [Ks[s] for s in act], sequences=act)
            n += len(act)
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def run_single(trks, frames, Ks, sched):
    """One num_sequences=1 tracker per stream, the active ones stepped back to back -> stream-frames/s."""
    for trk in trks:
        trk.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for t, act in enumerate(sched):
        for s in act:
            trks[s].step([frames[t][s]], [Ks[s]])
            n += 1
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def reserved():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return torch.cuda.memory_reserved()


def peak_since(base):
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_reserved() - base) / 2 ** 20


def replay_fps(ticks, reps=3):
    """ticks: per tick (stream-frames, [captured stages replayed that tick]) -> stream-frames/s of replaying them all."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _, sts in ticks[:3]:
        for st in sts:
            st.graph.replay()
    a.record()
    for _ in range(reps):
        for _, sts in ticks:
            for st in sts:
                st.graph.replay()
    b.record()
    torch.cuda.synchronize()
    return reps * sum(n for n, _ in ticks) / (a.elapsed_time(b) / 1e3)


def tick_stages(trk, frames, Ks, sched, single=False):
    """Step the schedule once, recording the captured graph of every step -> per tick (stream-frames, [stages])."""
    trks = trk if single else [trk]
    log = []
    for tk in trks:                                         # StageCache.run, also noting the stage it replayed
        def run(name, fn, inputs, cache=tk.stages, orig=tk.stages.run):
            out = orig(name, fn, inputs)
            log.append(cache.stages[(name,) + tuple((tuple(t.shape), t.dtype) for t in inputs)])
            return out
        tk.stages.run = run
    out = []
    for t, act in enumerate(sched):
        if not act:
            continue
        del log[:]
        if single:
            for s in act:
                trk[s].step([frames[t][s]], [Ks[s]])
        else:
            trk.step([frames[t][q] for q in act], [Ks[q] for q in act], sequences=act)
        out.append((len(act), list(log)))
    for tk in trks:
        del tk.stages.run
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='4,10')
    ap.add_argument('--T', type=int, default=60)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--refine-iter', type=int, default=1)
    args = ap.parse_args()
    est, db = syn.build_estimator()
    est.cfg['device_glue'] = True
    K = db.K
    med = lambda xs: round(float(np.median(xs)), 1)
    res = {}
    for S in [int(s) for s in args.S.split(',')]:
        videos = [[db.render(p, K) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), args.T)] for s in range(S)]
        frames = [[videos[s][t] for s in range(S)] for t in range(args.T)]
        Ks = [K] * S
        res[S] = {}
        for name in ('rates', 'drops', 'all'):
            sched = schedule(name, S, args.T)
            base = reserved()
            trk = est.tracker(num_sequences=S, refine_iter=args.refine_iter)
            ticks_p = tick_stages(trk, frames, Ks, sched)           # capture every graph the schedule needs
            mem_p = peak_since(base)
            base = reserved()
            singles = [est.tracker(num_sequences=1, refine_iter=args.refine_iter) for _ in range(S)]
            ticks_s = tick_stages(singles, frames, Ks, sched, single=True)
            mem_s = peak_since(base)
            e2e = {'partial': [], 'per_stream': []}
            dev = {'partial': [], 'per_stream': []}
            for _ in range(args.runs):
                e2e['partial'].append(run_partial(trk, frames, Ks, sched))
                e2e['per_stream'].append(run_single(singles, frames, Ks, sched))
                dev['partial'].append(replay_fps(ticks_p))
                dev['per_stream'].append(replay_fps(ticks_s))
            active = [len(a) for a in sched]
            res[S][name] = {
                'mean_active': round(float(np.mean(active)), 2),
                'e2e_fps': {k: med(v) for k, v in e2e.items()}, 'dev_fps': {k: med(v) for k, v in dev.items()},
                'graphs': {'partial': len(trk.stages.stages), 'per_stream': sum(len(t.stages.stages) for t in singles)},
                'kernels_per_graph': {'partial': sorted({st.kernels for st in trk.stages.stages.values()}),
                                      'per_stream': sorted({st.kernels for t in singles for st in t.stages.stages.values()})},
                'graph_memory_mb': {'partial': round(mem_p, 1), 'per_stream': round(mem_s, 1)}}
            print(json.dumps({'S': S, 'schedule': name, **res[S][name]}), file=sys.stderr, flush=True)
            del trk, singles, ticks_p, ticks_s
    # K = 2 objects at the largest S under 'rates'
    torch.cuda.empty_cache()
    S = max(int(s) for s in args.S.split(','))
    objs = est.object_set()
    for i, seed in enumerate((7, 8)):
        objs.add(f'o{i}', syn.synthetic_database(seed=seed))
    videos = [[db.render(p, K) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), args.T)] for s in range(S)]
    frames = [[videos[s][t] for s in range(S)] for t in range(args.T)]
    sched = schedule('rates', S, args.T)
    otrk = objs.tracker(num_sequences=S, refine_iter=args.refine_iter)
    osingles = [objs.tracker(num_sequences=1, refine_iter=args.refine_iter) for _ in range(S)]
    run_partial(otrk, frames, [K] * S, sched)                       # capture
    run_single(osingles, frames, [K] * S, sched)
    fps = {'partial': [], 'per_stream': []}
    for _ in range(args.runs):
        fps['partial'].append(run_partial(otrk, frames, [K] * S, sched) * len(objs))
        fps['per_stream'].append(run_single(osingles, frames, [K] * S, sched) * len(objs))
    res['objects_K2'] = {'S': S, 'schedule': 'rates', 'e2e_object_fps': {k: med(v) for k, v in fps.items()},
                         'graphs': {'partial': len(otrk.stages.stages), 'per_stream': sum(len(t.stages.stages) for t in osingles)}}
    name, plimit = card()
    print(json.dumps({'tool': 'partial_track_bench', 'gpu': name, 'power_limit_w': plimit, 'T': args.T, 'runs': args.runs,
                      'refine_iter': args.refine_iter, 'results': res}))


if __name__ == '__main__':
    main()
