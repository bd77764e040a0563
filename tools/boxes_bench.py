"""Boxes from another detector (row f19) against Gen6D's detector, on instance_track_bench.py's video (two translating
copies of the synthetic object at 480x640), cfg['refine_iter'] = 3.  The boxes are the detector's own records of an earlier
call made squares of side ref_resolution * scale, so both paths pose the same objects.  One JSON line with the card and
its power limit read in the same run; every rate the median of --repeats runs, the two paths alternating.
  (a) predict_batch at qn frames: poses/s device-resident (CUDA events around the graph replay) and end to end (host
      clock around the call, which ends in its synchronising read), kernels per graph, peak reserved MiB;
  (b) predict_instances at M = 1 and 4 on the same frames: instance-poses/s (M * qn per call), kernels, peak MiB;
  (c) est.instance_tracker(max_instances=2) at S sequences, T steps: 'detector' (redetect_every = E), 'boxes_every_E'
      (redetect_every = None, boxes on every E-th step) and 'boxes_every_step': instance-frames/s (M * S per step) end to
      end and device-resident, peak MiB.
  python tools/boxes_bench.py [--qn 10] [--S 4,10] [--E 10] [--T 40] [--repeats 3] [--dry-run]"""
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
    ap.add_argument('--qn', type=int, default=10)
    ap.add_argument('--S', default='4,10', help='comma-separated sequence counts')
    ap.add_argument('--E', type=int, default=10, help='re-detection period')
    ap.add_argument('--T', type=int, default=40, help='frames per video')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--dry-run', action='store_true', help='check the arguments and print the plan, no GPU needed')
    args = ap.parse_args(argv)
    try:
        args.S = sorted({int(s) for s in args.S.split(',')})
    except ValueError:
        ap.error('--S takes comma-separated integers')
    if args.qn < 1 or min(args.S) < 1 or args.E < 1 or args.T < 2 or args.repeats < 1:
        ap.error('need qn, S, E, repeats >= 1 and T >= 2')
    return args


def squares(inter, f, M=None):
    """The valid detection records of frame f of an inter (predict_instances' keys, or predict_batch's when M is None)
    -> boxes float32 [n, 5]: the square of side 128 * scale at the detected position, with the detection score."""
    import numpy as np
    if M is None:
        x, y = inter['det_position'][f]
        s = inter['det_scale_r2q'][f]
        return np.float32([[x - 64 * s, y - 64 * s, x + 64 * s, y + 64 * s, 1.0]])
    keep = inter['instance_valid'][f]
    (x, y), s, sc = inter['det_position'][f, keep].T, inter['det_scale_r2q'][f, keep], inter['det_score'][f, keep]
    return np.stack([x - 64 * s, y - 64 * s, x + 64 * s, y + 64 * s, sc], 1).astype(np.float32)


def main():
    args = parse()
    if args.dry_run:
        print(json.dumps({'tool': 'boxes_bench', 'dry_run': True, 'qn': args.qn, 'S': args.S, 'E': args.E, 'T': args.T,
                          'repeats': args.repeats}))
        return
    import torch
    from gen6d_b200 import synthetic as syn
    from gen6d_b200.graphs import CapturedStage
    from instance_track_bench import video
    from track_bench import card

    db = syn.synthetic_database(seed=7)
    est = syn.build_estimator(db)[0]
    assert est.cfg['refine_iter'] == 3
    T, E, qn = args.T, args.E, args.qn
    seqs = [video(db, T, -8.0 * s) for s in range(max(max(args.S), 1))]
    assert seqs[0][0][0].shape == (480, 640, 3), seqs[0][0][0].shape
    med = statistics.median

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

    def release(*owners):
        for o in set(owners) | {est}:
            o.stages.clear()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()

    def timed(fn, n_calls):
        """n_calls calls of fn -> (wall seconds, device seconds)."""
        events.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n_calls):
            fn(i)
        wall = time.perf_counter() - t0
        return wall, sum(a.elapsed_time(b) for a, b in events) / 1e3

    def compare(variants, work, n_calls):
        """variants {name: fn(i)}, alternating, run 0 a warm-up -> {name: {e2e, dev, kernels, peak_mib}}."""
        stats = {v: {'e2e': [], 'dev': []} for v in variants}
        for rep in range(args.repeats + 1):
            for v, fn in variants.items():
                wall, dev = timed(fn, n_calls)
                if rep:
                    stats[v]['e2e'].append(work / wall)
                    stats[v]['dev'].append(work / dev)
        return {v: {'e2e': round(med(s['e2e']), 1), 'dev': round(med(s['dev']), 1)} for v, s in stats.items()}

    def single(fn, owner):
        """Kernels per graph and peak reserved MiB of one variant run on its own from an empty graph cache."""
        release(owner)
        fn(0)
        torch.cuda.synchronize()
        return {'kernels': sorted({st.kernels for st in owner.stages.stages.values()}),
                'peak_mib': round(torch.cuda.max_memory_reserved() / 2 ** 20, 1)}

    name, power = card()
    res = {'tool': 'boxes_bench', 'card': name, 'power_limit_w': power, 'qn': qn, 'refine_iter': est.cfg['refine_iter']}
    imgs = [seqs[i % len(seqs)][0][i // len(seqs)] for i in range(qn)]
    Ks = [seqs[i % len(seqs)][1] for i in range(qn)]

    # (a) predict_batch
    _, inter = est.predict_batch(imgs, Ks)
    one = [squares(inter, f) for f in range(qn)]
    variants = {'detector': lambda i: est.predict_batch(imgs, Ks), 'boxes': lambda i: est.predict_batch(imgs, Ks, boxes=one)}
    row = compare(variants, qn * 5, 5)
    for v, fn in variants.items():
        row[v].update(single(fn, est))
    res['predict_batch'] = row

    # (b) predict_instances
    res['predict_instances'] = []
    for M in (1, 4):
        _, inter = est.predict_instances(imgs, Ks, max_instances=M)
        bx = [squares(inter, f, M) for f in range(qn)]
        variants = {'detector': lambda i, M=M: est.predict_instances(imgs, Ks, max_instances=M),
                    'boxes': lambda i, M=M, bx=bx: est.predict_instances(imgs, Ks, max_instances=M, boxes=bx)}
        row = compare(variants, qn * M * 5, 5)
        for v, fn in variants.items():
            row[v].update(single(fn, est))
        res['predict_instances'].append({'M': M, **row})
    release()

    # (c) instance trackers
    res['instance_tracker'] = []
    M = 2
    for S in args.S:
        Kseq = [seqs[s][1] for s in range(S)]
        frames = [[seqs[s][0][t] for s in range(S)] for t in range(T)]
        boxes = []
        for t in range(T):
            _, inter = est.predict_instances(frames[t], Kseq, max_instances=M)
            boxes.append([squares(inter, s, M) for s in range(S)])
        release()
        trks = {'detector': est.instance_tracker(num_sequences=S, max_instances=M, redetect_every=E),
                f'boxes_every_{E}': est.instance_tracker(num_sequences=S, max_instances=M),
                'boxes_every_step': est.instance_tracker(num_sequences=S, max_instances=M)}

        def run(v, trk):
            def video_run(_):
                trk.reset()
                for t in range(T):
                    if v == 'detector':
                        trk.step(frames[t], Kseq)
                    elif v == 'boxes_every_step' or t % E == 0:
                        trk.step(frames[t], Kseq, boxes=boxes[t])
                    else:
                        trk.step(frames[t], Kseq)
            return video_run
        variants = {v: run(v, trk) for v, trk in trks.items()}
        row = compare(variants, T * S * M, 1)
        for v, fn in variants.items():
            row[v].update(single(fn, trks[v]))
        res['instance_tracker'].append({'S': S, 'M': M, 'T': T, **row})
        release(*trks.values())
    CapturedStage.__call__ = orig_call
    print(json.dumps(res))


if __name__ == '__main__':
    main()
