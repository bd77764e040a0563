"""Cost of checking the instance trackers' tracks with the detector (row f21), with the card and its power limit read in
the same run.  tools/instance_track_bench.py's video (T frames at 480x640, two copies of the synthetic object translating
across the frame), M = 2 slots, lockstep, refine_iter = 1, T steps from a reset.
  * per S and schedule (detect once; redetect_every 5 / 10; verify_every 5 / 10 with no threshold, detected once):
    instance-frames/s (M slots x S sequences per step) end to end (trk.step on numpy frames) and device-resident (the
    step graphs that ran, replayed in the same order on the device-held inputs, CUDA events), medians of three alternating
    runs; kernels per graph; peak reserved memory.
The checkpoint is random: scores say nothing about how well losses are caught, so no threshold is set and the numbers are
costs only.
  python tools/instance_verify_bench.py [--S 1,4,10] [--T 40]"""
import argparse
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from gen6d_b200 import synthetic as syn  # noqa: E402
from instance_track_bench import video  # noqa: E402
from track_bench import card  # noqa: E402
from verify_bench import kernels, measure  # noqa: E402

M = 2
# (name, redetect_every, verify_every)
SCHEDULES = [('detect_once', None, None), ('redetect5', 5, None), ('redetect10', 10, None), ('verify5', None, 5),
             ('verify10', None, 10)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--S', default='1,4,10')
    ap.add_argument('--T', type=int, default=40)
    args = ap.parse_args()
    est, db = syn.build_estimator()
    T = args.T
    out = {}
    for S in [int(s) for s in args.S.split(',')]:
        clips = [video(db, T, 10.0 * s) for s in range(S)]
        frames, Ks = [[clips[s][0][t] for s in range(S)] for t in range(T)], [clips[s][1] for s in range(S)]
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        plain = {E: est.instance_tracker(S, max_instances=M, redetect_every=E) for E in (None, 5, 10)}
        checking = est.instance_tracker(S, max_instances=M, verify_every=1)
        # verify_bench.measure's run(reset_every=None) keeps the tracker's own schedule; the verifying schedules share one
        # tracker whose verify_every is set before each run
        trackers = {name: (checking if every else plain[E], every, None) for name, E, every in SCHEDULES}
        fps = measure(trackers, frames, Ks, M * S * T)
        res = {name: {'e2e_ifps': round(e, 1), 'dev_ifps': round(d, 1)} for name, (e, d) in fps.items()}
        res['kernels'] = {'plain': kernels(plain[5]), 'verifying': kernels(checking)}
        res['peak_reserved_mb'] = round(torch.cuda.max_memory_reserved() / 2 ** 20)
        out[S] = res
        print(json.dumps({'S': S, **res}), file=sys.stderr, flush=True)
        del plain, checking, trackers
    name, plimit = card()
    print(json.dumps({'tool': 'instance_verify_bench', 'gpu': name, 'power_limit_w': plimit, 'M': M, 'T': T, 'results': out}))


if __name__ == '__main__':
    main()
