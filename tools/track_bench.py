"""Tracking throughput: S sequences x T rendered frames through Gen6DEstimator.tracker (device-glue path), one JSON line
with the card and its power limit read in the same run.
  * track_dev_fps: tracked frames/s, device-resident (the refine-step graph replayed on frames already on the device);
  * track_e2e_fps: tracked frames/s end to end (trk.step with numpy frames: upload, one replay, one read, unpack);
  * step_ms: mean end-to-end step time;
  * predict_batch_fps: predict_batch (device glue) poses/s at the same S, for comparison.
  python tools/track_bench.py [--S 1,4,10] [--T 40]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen6d_b200 import synthetic as syn  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return name, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='1,4,10')
    ap.add_argument('--T', type=int, default=40)
    args = ap.parse_args()
    est, db = syn.build_estimator()
    K = db.K
    # a smooth camera path around a database view (tests/golden/track_cases.track_case)
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
    from golden import track_cases
    res = {}
    for S in [int(s) for s in args.S.split(',')]:
        videos = [[db.render(p, K) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), args.T)] for s in range(S)]
        frames = [[videos[s][t] for s in range(S)] for t in range(args.T)]
        Ks = [K] * S
        trk = est.tracker(num_sequences=S)
        for t in range(3):                                      # warm-up: capture the full and the refine graphs
            trk.step(frames[t], Ks)
        trk.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(args.T):
            trk.step(frames[t], Ks)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
        # steady state: time only the tracked (refine-only) steps
        t0 = time.perf_counter()
        for t in range(1, args.T):
            trk.step(frames[t], Ks)
        torch.cuda.synchronize()
        e2e_refine = time.perf_counter() - t0
        # device-resident: replay the refine step's graph on frames already uploaded
        stage = [s for k, s in trk.stages.stages.items() if k[0].startswith('track_refine')][0]
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            stage.graph.replay()
        start.record()
        for _ in range(args.T):
            stage.graph.replay()
        stop.record()
        torch.cuda.synchronize()
        dev_s = start.elapsed_time(stop) / 1e3
        # predict_batch at the same S
        est.predict_batch(frames[0], Ks)
        torch.cuda.synchronize()
        n_pb = max(4, args.T // 4)
        t0 = time.perf_counter()
        for t in range(n_pb):
            est.predict_batch(frames[t], Ks)
        torch.cuda.synchronize()
        pb = time.perf_counter() - t0
        res[S] = {'track_dev_fps': round(S * args.T / dev_s, 1), 'track_e2e_fps': round(S * (args.T - 1) / e2e_refine, 1),
                  'step_ms': round(e2e_refine / (args.T - 1) * 1e3, 3), 'dev_step_ms': round(dev_s / args.T * 1e3, 3),
                  'e2e_fps_with_first_frame': round(S * args.T / e2e, 1), 'predict_batch_fps': round(S * n_pb / pb, 1)}
        print(json.dumps({'S': S, **res[S]}), file=sys.stderr, flush=True)
    name, plimit = card()
    print(json.dumps({'tool': 'track_bench', 'gpu': name, 'power_limit_w': plimit, 'T': args.T, 'results': res}))


if __name__ == '__main__':
    main()
