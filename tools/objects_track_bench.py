"""Tracking an object set: ObjectSet.tracker (one refine-step graph over all K objects, object-indexed glue and
smoothing launches, one refiner stage over K*S poses) against K one-object sets' trackers stepped back to back.  A
one-object set's tracker is bit-identical to est.tracker() (tests/test_track_objects_gpu.py), so it stands in for K
estimators without K copies of the networks.  One JSON line with the card and its power limit read in the same run.

For each K (synthetic objects of seeds 7, 8, ...) and S (sequences in lockstep), T frames rendered along
tests/golden/track_cases.track_case from the first object's database.  The frames' content does not change the work of a
tracked step (the same crops, refiner and PnP run whatever the frames show), so every object is tracked on them.
  * set_dev / sep_dev: tracked object-frames/s device-resident (the refine-step graphs replayed on frames already on the
    device; the K separate trackers are timed one after the other and their times summed, since every step ends in a
    synchronising read);
  * set_e2e / sep_e2e: tracked object-frames/s end to end (step() on numpy frames: upload, one replay, one read, unpack);
  * set_kernels / sep_kernels: kernels of the set's refine-step graph / of the K separate refine-step graphs together;
each the median of --repeats runs, the two variants alternating; the graphs of one configuration are freed before the
next.  A configuration that does not fit in memory is
recorded as such.
  python tools/objects_track_bench.py [--K 1,2,4,8] [--S 1,4,10] [--T 40] [--repeats 3]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', default='1,2,4,8')
    ap.add_argument('--S', default='1,4,10')
    ap.add_argument('--T', type=int, default=40)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    from gen6d_b200 import synthetic as syn
    from golden import track_cases
    from track_bench import card

    Kmax = max(int(k) for k in args.K.split(','))
    dbs = [syn.synthetic_database(seed=7 + k) for k in range(Kmax)]
    est = syn.build_estimator(dbs[0])[0]
    est.cfg['device_glue'] = True
    db, Kcam = dbs[0], dbs[0].K

    def release(*trackers):
        for t in trackers:
            t.stages.clear()
        gc.collect()
        torch.cuda.empty_cache()

    def refine_stage(trk):
        return [s for k, s in trk.stages.stages.items() if k[0].startswith('track_refine')][0]

    def warm(trk, frames, Ks):
        """A full step and two refine steps capture both graphs; the full one is freed (only refine steps are timed)."""
        for t in range(3):
            trk.step(frames[t], Ks)
        for k in [k for k in trk.stages.stages if k[0] == 'track_full']:
            del trk.stages.stages[k]
        torch.cuda.synchronize()
        return refine_stage(trk)

    def e2e(trk, frames, Ks):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(1, args.T):
            trk.step(frames[t], Ks)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / (args.T - 1)

    def dev(stage):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            stage.graph.replay()
        start.record()
        for _ in range(args.T):
            stage.graph.replay()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / 1e3 / args.T

    Ks_list = [int(k) for k in args.K.split(',')]
    sets = {}                           # K -> a set of the first K objects
    for K in Ks_list:
        sets[K] = est.object_set()
        for k in range(K):
            sets[K].add(f'obj{k}', dbs[k])
    ones = [est.object_set() for _ in range(Kmax)]
    for k, one in enumerate(ones):
        one.add(f'obj{k}', dbs[k])
    res = {}
    for S in [int(s) for s in args.S.split(',')]:
        videos = [[db.render(p, Kcam) for p in track_cases.track_case(db.get_pose(str(11 + 3 * s)), args.T)] for s in range(S)]
        frames = [[videos[s][t] for s in range(S)] for t in range(args.T)]
        Ks = [Kcam] * S
        for K in Ks_list:
            key = f'K{K}_S{S}'
            trackers = []
            try:
                trk = sets[K].tracker(num_sequences=S)
                trackers.append(trk)
                stage = warm(trk, frames, Ks)
                seps = []
                for one in ones[:K]:
                    t1 = one.tracker(num_sequences=S)
                    trackers.append(t1)
                    seps.append((t1, warm(t1, frames, Ks)))
                runs = {'set_dev': [], 'sep_dev': [], 'set_e2e': [], 'sep_e2e': []}
                for _ in range(args.repeats):
                    runs['set_dev'].append(K * S / dev(stage))
                    runs['set_e2e'].append(K * S / e2e(trk, frames, Ks))
                    runs['sep_dev'].append(K * S / sum(dev(st) for _, st in seps))
                    runs['sep_e2e'].append(K * S / sum(e2e(t1, frames, Ks) for t1, _ in seps))
                res[key] = {k: round(statistics.median(v), 1) for k, v in runs.items()}
                res[key].update(runs={k: [round(x, 1) for x in v] for k, v in runs.items()}, set_kernels=stage.kernels,
                                sep_kernels=sum(st.kernels for _, st in seps),
                                set_dev_step_ms=round(1e3 * K * S / res[key]['set_dev'], 3),
                                sep_dev_step_ms=round(1e3 * K * S / res[key]['sep_dev'], 3),
                                peak_reserved_gb=round(torch.cuda.max_memory_reserved() / 2 ** 30, 1))
                del stage, seps
            except torch.cuda.OutOfMemoryError:
                res[key] = 'out of memory'
            release(*trackers)
            del trackers
            print(json.dumps({key: res[key]}), file=sys.stderr, flush=True)
    name, plimit = card()
    print(json.dumps({'tool': 'objects_track_bench', 'gpu': name, 'power_limit_w': plimit, 'T': args.T, 'repeats': args.repeats,
                      'unit': 'tracked object-frames/s', 'results': res}))


if __name__ == '__main__':
    main()
