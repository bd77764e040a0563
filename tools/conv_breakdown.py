"""Time / TFLOP/s of every tensor-core convolution in one batched pose step, per shape.

    python tools/conv_breakdown.py [--batch B] [--refine-iter N] [--reps C] [--repeat R]

The stages of one `predict_batch` over B synthetic frames (detect -> select -> N refinements; bench.py's
workload is B = 10, N = 3) are recorded with their device inputs and replayed once eagerly to collect the
arguments of every convolution.  Each distinct call is then timed on its own: a CUDA graph of C copies of
it, replayed R times, median per copy (timing the calls inside the eager replay would measure the host
whenever a kernel is shorter than its launch).  Each line aggregates the calls of one tag; the tag names
the kernel the planner picked (persist: the persistent kernel, reuse: the A-reuse kernel), the prologue,
BN, the K splits and how a persistent call gets its A operand (im2col: by TMA from a split copy of the input,
prenorm: the same from a copy with the prologue applied; neither: gathered by the producer warps; a '-ro' suffix
marks a layer the A-reuse kernel would take, run in its K order by G6D_TC_REUSE_IM2COL; 'fold' marks K splits summed in
the output by G6D_TC_FOLD_SPLITS instead of through fp32 partials and a reduce pass).  Times are per step of B
poses, split pass included.  Class lines sum the calls of each part of the network (detector correlation, the
crops' VGG, selector towers, ...; see CLASSES) and list those of its tags that plan the A-reuse kernel or were taken
from it."""
import argparse
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen6d_b200 import ops, synthetic as syn  # noqa: E402


def record_step(batch, refine_iter):
    """(estimator, [(stage fn, inputs)]) of one predict_batch over `batch` frames."""
    est, db = syn.build_estimator(refine_iter=refine_iter)
    ids = db.get_img_ids()
    imgs = [db.get_image(ids[(7 + 3 * i) % len(ids)]) for i in range(batch)]
    rec, mods = [], [m for m in (est, est.detector, est.selector, est.refiner) if m is not None]
    for m in mods:
        def wrapped(name, fn, inputs, _o=m.stages.run):
            rec.append((fn, list(inputs)))
            return _o(name, fn, inputs)
        m.stages.run = wrapped
    try:
        est.predict_batch(imgs, [db.K] * batch)
    finally:
        for m in mods:
            del m.stages.run
    torch.cuda.synchronize()
    return est, rec


# (class, method name, label): each ops.conv call is labelled by the innermost of these methods it runs under
CLASSES = (
    ('Detector', '_detect_maps', 'detector heads'),
    ('Detector', '_features', 'detector VGG'),
    ('Detector', '_raw_correlation', 'detector correlation'),
    ('Detector', '_raw_correlation_objects', 'detector correlation'),
    ('ViewpointSelector', '_select_chunk', 'selector 1x1 layers'),
    ('ViewpointSelector', '_feats', 'selector crop VGG'),
    ('ViewpointSelector', '_tower_conv', 'selector towers'),
    ('VolumeRefiner', '_feature_net', 'refiner crop VGG'),
    ('VolumeRefiner', '_volume_net', 'refiner volume net + feature branches'),
    ('VolumeRefiner', '_conv_in_conv', 'refiner volume net + feature branches'),
)


def conv_calls(rec):
    """(args, kwargs, label) of every ops.conv call of one eager replay of the recorded stages (the tensors stay
    alive).  The label is that of the innermost method of CLASSES the call runs under ('other' outside them)."""
    from gen6d_b200.network import detector, refiner, selector
    owners = {'Detector': detector.Detector, 'ViewpointSelector': selector.ViewpointSelector,
              'VolumeRefiner': refiner.VolumeRefiner}
    calls, orig, stack = [], ops.conv, ['other']
    saved = [(owners[c], n, getattr(owners[c], n), label) for c, n, label in CLASSES]

    def wrapped(*a, **k):
        calls.append((a, k, stack[-1]))
        return orig(*a, **k)

    def marking(f, label):
        def g(*a, **k):
            stack.append(label)
            try:
                return f(*a, **k)
            finally:
                stack.pop()
        return g
    ops.conv = wrapped
    for cls, n, f, label in saved:
        setattr(cls, n, marking(f, label))
    try:
        with torch.no_grad():
            for fn, inputs in rec:
                fn(*inputs)
    finally:
        ops.conv = orig
        for cls, n, f, _ in saved:
            setattr(cls, n, f)
    torch.cuda.synchronize()
    return calls


def time_call(a, k, reps, repeat):
    """(tag, flop, ms) of one tensor-core ops.conv call: the median over `repeat` replays of a graph of `reps`
    back-to-back copies of the call, per copy.  None for a call that does not take the tensor-core path."""
    prof = ops.enable_profiling()
    ops.conv(*a, **k)
    calls = ops.collect_profile(prof).get('#calls')
    if not calls:
        return None
    _, work, _, tag = calls[0]
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        for _ in range(reps):
            ops.conv(*a, **k)
    g.replay()
    times = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / reps)
    del g
    return tag, work, sorted(times)[len(times) // 2]


def breakdown(calls, reps=10, repeat=5):
    """({tag: [calls, ms, flop]} per step, {label: {tag: [calls, ms, flop]}}).  Calls with the same tag are timed
    once (the first of them)."""
    agg, timed, labels = collections.OrderedDict(), {}, collections.OrderedDict()
    for a, k, label in calls:
        prof = ops.enable_profiling()
        ops.conv(*a, **k)
        c = ops.collect_profile(prof).get('#calls')
        if not c:
            continue
        tag = c[0][3]
        if tag not in timed:
            timed[tag] = time_call(a, k, reps, repeat)
        _, work, ms = timed[tag]
        for e in (agg.setdefault(tag, [0, 0.0, 0.0]), labels.setdefault(label, {}).setdefault(tag, [0, 0.0, 0.0])):
            e[0] += 1; e[1] += ms; e[2] += work
    return agg, labels


def no_prologue_3x3_persistent(tag):
    """The layers whose A operand could come from a split activation: stride-1 3x3, no prologue, persistent kernel."""
    return ' k=1x3x3 s=1 pro=0 persist ' in f' {tag} '


def prologue_3x3_persistent(tag):
    """The layers a prologue-applied split input can feed (the selector towers' 8x8 and 4x4 layers), whichever way
    they ran: stride-1 3x3 with a prologue on the persistent kernel."""
    return ' k=1x3x3 s=1 pro=' in f' {tag} ' and ' pro=0 ' not in f' {tag} ' and ' persist ' in f' {tag} '


def folded_partial_bytes(tag):
    """The fp32 split-K partials (splits x M x N) a call tagged 'fold' no longer writes; 0 for other calls."""
    if ' fold' not in tag:
        return 0
    f = dict(t.split('=', 1) for t in tag.split() if t.startswith(('M=', 'N=', 'splits=')))
    return 4 * int(f['splits']) * int(f['M']) * int(f['N'])


def report(agg, labels, top=40):
    tot_ms, tot_w = sum(a[1] for a in agg.values()), sum(a[2] for a in agg.values())
    print(f'conv_tc calls {sum(a[0] for a in agg.values())} total {tot_ms:.2f} ms, {tot_w / tot_ms / 1e9:.1f} TFLOP/s')
    classes = collections.OrderedDict()
    for tag, (n, ms, w) in agg.items():
        key = ' '.join(t for t in tag.split() if t.startswith(('pro=', 'persist', 'reuse', 'fold', 'prenorm', 'im2col')))
        c = classes.setdefault(key, [0, 0.0, 0.0]); c[0] += n; c[1] += ms; c[2] += w
    for key, (n, ms, w) in sorted(classes.items(), key=lambda kv: -kv[1][1]):
        print(f'  {ms:7.3f} ms x{n:3d} {w / ms / 1e9:6.1f} TF/s  [{key}]')
    for what, pick in (('3x3 stride 1, no prologue, persistent', no_prologue_3x3_persistent),
                       ('3x3 stride 1, prologue, persistent', prologue_3x3_persistent)):
        sel = [a for t, a in agg.items() if pick(t)]
        if sel:
            ms, w = sum(a[1] for a in sel), sum(a[2] for a in sel)
            print(f'  {ms:7.3f} ms x{sum(a[0] for a in sel):3d} {w / ms / 1e9:6.1f} TF/s  [{what}]')
    for label, tags in labels.items():
        n, ms, w = (sum(a[i] for a in tags.values()) for i in range(3))
        print(f'  {ms:7.3f} ms x{n:3d} {w / ms / 1e9:6.1f} TF/s  [{label}, {100 * ms / tot_ms:.1f} % of the total]')
        saved = sum(a[0] * folded_partial_bytes(t) for t, a in tags.items())
        if saved:
            print(f'      fold: {saved / 1e9:.2f} GB of fp32 partials not written (nor read back by a reduce pass)')
        for tag, (n, ms, w) in sorted(tags.items(), key=lambda kv: -kv[1][1]):
            if ' reuse ' in f' {tag} ' or tag.endswith('-ro'):
                print(f'      {ms:7.3f} ms x{n:3d} {w / ms / 1e9:6.1f} TF/s  {tag}')
    for tag, (n, ms, w) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
        print(f'{ms:7.3f} ms x{n:3d} {w / ms / 1e9:6.1f} TF/s  {tag}')


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--batch', type=int, default=10, help='frames per predict_batch (bench.py: 10)')
    ap.add_argument('--refine-iter', type=int, default=3, help='refinements per pose (bench.py: 3)')
    ap.add_argument('--reps', type=int, default=10, help='copies of a call per captured graph')
    ap.add_argument('--repeat', type=int, default=5, help='timed graph replays per call (median)')
    ap.add_argument('--top', type=int, default=40, help='shapes listed')
    a = ap.parse_args()
    ops.require_cuda()
    _, rec = record_step(a.batch, a.refine_iter)
    print(f'{torch.cuda.get_device_name()}: batch {a.batch}, {a.refine_iter} refinements, '
          f'median of {a.repeat} replays of {a.reps} copies per shape')
    report(*breakdown(conv_calls(rec), a.reps, a.repeat), top=a.top)


if __name__ == '__main__':
    main()
