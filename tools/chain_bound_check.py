"""Cost and benefit of the tensor-core accumulate-chain bound (conv_tc.cu: every convolution with K > 2048 is
split into 2048-element chains summed in fp32 round-to-nearest).  Runs the detector at full size (480x640 frame,
32 reference views, tests/golden/det32_golden.npz) twice: with the bound, and with every convolution of
K <= 8192 left in one chain (its max_chain_k set to K).  For each it prints the raw correlation's error against
the reference's golden values and the time of one detection (CUDA events, median of 10 after 3 warm-ups).

    python tools/chain_bound_check.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from golden import cases  # noqa: E402
from gen6d_b200 import ops  # noqa: E402
from test_networks_gpu import HERE, build, sub, to_nchw  # noqa: E402


def packed_convs(obj, seen=None):
    """Every ops.PackedConv reachable from obj's attributes, lists, tuples and dicts."""
    seen = set() if seen is None else seen
    if id(obj) in seen:
        return []
    seen.add(id(obj))
    if isinstance(obj, ops.PackedConv):
        return [obj]
    if isinstance(obj, (list, tuple)):
        items = obj
    elif isinstance(obj, dict):
        items = obj.values()
    elif type(obj).__module__.startswith(('gen6d_b200', 'torch.nn')) and hasattr(obj, '__dict__'):
        items = vars(obj).values()
    else:
        return []
    return [pc for it in items for pc in packed_convs(it, seen)]


def measure(net, que01, D):
    with torch.no_grad():
        o = net._detect_nhwc(que01, return_taps=True)
        rel, signed = [], []
        for si, per_scale in enumerate(o['raw']):
            for l, raw in enumerate(per_scale):
                g, want = sub(to_nchw(raw)).astype(np.float64), D[f'raw.s{si}.l{l}.sub'].astype(np.float64)
                big = np.abs(want) > 1e3
                rel.append(np.abs(g - want)[big] / np.abs(want)[big])
                signed.append(((g - want) / want)[big])
        rel, signed = np.concatenate(rel), np.concatenate(signed)
        for _ in range(3):
            net._detect_nhwc(que01)
        times = []
        for _ in range(10):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            net._detect_nhwc(que01)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
    return {'max_rel_err': float(rel.max()), 'mean_signed_rel_err': float(signed.mean()),
            'share_beyond_3e-5': float((rel > 3e-5).mean()), 'detect_ms': float(np.median(times))}


def main():
    D = np.load(os.path.join(HERE, 'golden', 'det32_golden.npz'))
    c = cases.detector_case_full()
    net, _ = build('detector', {'name': 'det', 'network': 'detector', **c['cfg']})
    net.load_ref_imgs(c['ref_imgs'])
    que01 = ops.preprocess_u8(torch.from_numpy(c['que_imgs']).cuda(), out_c=3, imagenet_norm=False)
    out = {'bounded (K > 2048 split)': measure(net, que01, D)}
    convs = packed_convs(net)
    unsplit = [pc for pc in convs if pc.max_chain_k == 0 and 2048 < pc.cin * int(np.prod(pc.k)) <= 8192]
    for pc in unsplit:
        pc.max_chain_k = pc.cin * int(np.prod(pc.k))
    out['unbounded for K <= 8192'] = measure(net, que01, D)
    out['convolutions affected'] = len(unsplit)
    out['gpu'] = torch.cuda.get_device_name()
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
