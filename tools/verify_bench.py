"""Cost of checking tracked poses with the detector (row f20), with the card and its power limit read in the same run.
tools/track_bench.py's 480x640 rendered camera paths, T steps from a full prediction, tracker refine_iter = 1.
  * per S and schedule (verify_every None / 1 / 5 / 10, or a blind reset() every 5 / 10 steps): tracked frames/s end to
    end (trk.step on numpy frames) and device-resident (the step graphs that run replayed in the same order on the
    device-held inputs, CUDA events), medians of three alternating runs; kernels per graph; peak reserved memory;
  * verify_poses alone for n = 1 / 4 / 10, CUDA events over graph replays;
  * objs.tracker() with K = 2 objects at S = 4.
The checkpoint is random: scores and thresholds say nothing about detection quality, so no threshold is set.
  python tools/verify_bench.py [--T 40]"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from gen6d_b200 import synthetic as syn, verify as V  # noqa: E402
from gen6d_b200.graphs import CapturedStage  # noqa: E402
from track_bench import card  # noqa: E402

SCHEDULES = [('none', None, None), ('verify1', 1, None), ('verify5', 5, None), ('verify10', 10, None),
             ('reset5', None, 5), ('reset10', None, 10)]


class Recorder:
    """Records the captured stages replayed while active."""

    def __enter__(self):
        self.stages, self._orig = [], CapturedStage.__call__
        rec = self

        def call(stage, *a):
            rec.stages.append(stage)
            return rec._orig(stage, *a)
        CapturedStage.__call__ = call
        return self

    def __exit__(self, *exc):
        CapturedStage.__call__ = self._orig


def run(trk, frames, Ks, reset_every):
    """One tracked run of T steps from a reset -> (seconds, the stages replayed)."""
    trk.reset()
    torch.cuda.synchronize()
    with Recorder() as rec:
        t0 = time.perf_counter()
        for t in range(len(frames)):
            if reset_every and t and t % reset_every == 0:
                trk.reset()
            trk.step(frames[t], Ks)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, rec.stages


def replay(stages):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for s in stages:
        s.graph.replay()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / 1e3


def measure(trackers, frames, Ks, n):
    """trackers {schedule: (tracker, verify_every, reset_every)} -> {schedule: (median end-to-end, median device-resident
    frames/s)} over three alternating runs.  Schedules share a tracker (and its graphs) where they replay the same graphs:
    the verifying ones differ only in verify_every, set before each run."""
    def go(trk, every, reset_every):
        if every is not None:
            trk._verify = V.Schedule(every)
        return run(trk, frames, Ks, reset_every)
    for args in trackers.values():                              # warm-up: capture every graph each schedule replays
        go(*args)
    times = {name: ([], []) for name in trackers}
    for _ in range(3):
        for name, args in trackers.items():
            secs, stages = go(*args)
            times[name][0].append(n / secs)
            times[name][1].append(n / replay(stages))
    return {name: (statistics.median(e), statistics.median(d)) for name, (e, d) in times.items()}


def kernels(trk):
    return {str(k[0]): s.kernels for k, s in trk.stages.stages.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='1,4,10')
    ap.add_argument('--T', type=int, default=40)
    args = ap.parse_args()
    from golden import track_cases
    est, db = syn.build_estimator()
    K, T = db.K, args.T

    def video(S, dbs=(db,)):
        paths = [track_cases.track_case(db.get_pose(str(11 + 3 * s)), T) for s in range(S)]
        return [[dbs[s % len(dbs)].render(paths[s][t], K) for s in range(S)] for t in range(T)]
    out = {'tracker': {}, 'verify_poses': {}, 'object_tracker': {}}
    for S in [int(s) for s in args.S.split(',')]:
        frames, Ks = video(S), [K] * S
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        plain, checking = est.tracker(S), est.tracker(S, verify_every=1)
        trackers = {name: (checking if every else plain, every, reset) for name, every, reset in SCHEDULES}
        fps = measure(trackers, frames, Ks, S * T)
        res = {name: {'e2e_fps': round(e, 1), 'dev_fps': round(d, 1)} for name, (e, d) in fps.items()}
        res['kernels'] = {'plain': kernels(plain), 'verifying': kernels(checking)}
        res['peak_reserved_mb'] = round(torch.cuda.max_memory_reserved() / 2 ** 20)
        out['tracker'][S] = res
        print(json.dumps({'S': S, **res}), file=sys.stderr, flush=True)
        del plain, checking, trackers
    for n in (1, 4, 10):
        frames, Ks = video(n)[0], [K] * n
        poses, _ = est.predict_batch(frames, Ks)
        est.verify_poses(frames, Ks, poses)
        stage = [s for k, s in est.stages.stages.items() if k[0][0] == 'verify_poses' and k[1][0][0] == n][0]
        replay([stage] * 3)
        dt = statistics.median(replay([stage] * 20) / 20 for _ in range(3))
        out['verify_poses'][n] = {'ms': round(dt * 1e3, 3), 'kernels': stage.kernels}
        print(json.dumps({'verify_poses_n': n, **out['verify_poses'][n]}), file=sys.stderr, flush=True)
    gc.collect()
    torch.cuda.empty_cache()
    db_b = syn.synthetic_database(seed=8)
    objs = est.object_set()
    objs.add('a', db)
    objs.add('b', db_b)
    S = 4
    frames, Ks = video(S, (db, db_b)), [K] * S
    plain, checking = objs.tracker(S), objs.tracker(S, verify_every=1)
    fps = measure({'none': (plain, None, None), 'verify5': (checking, 5, None), 'verify1': (checking, 1, None)}, frames, Ks,
                  2 * S * T)
    out['object_tracker'] = {name: {'e2e_poses_per_s': round(e, 1), 'dev_poses_per_s': round(d, 1)} for name, (e, d) in fps.items()}
    print(json.dumps({'object_tracker_K2_S4': out['object_tracker']}), file=sys.stderr, flush=True)
    name, plimit = card()
    print(json.dumps({'tool': 'verify_bench', 'gpu': name, 'power_limit_w': plimit, 'T': T, 'results': out}))


if __name__ == '__main__':
    main()
