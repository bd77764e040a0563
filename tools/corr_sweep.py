"""Detector correlation shapes (refs as kernels, Cout = 32): default tensor-core kernel vs the A-reuse
ROW mode (G6D_CONV_FLAT=2).  Spawns one process per setting (the switch is read once per process)."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SHAPES = [(88, 116, 15), (60, 80, 15), (44, 60, 15), (32, 40, 15), (44, 58, 7), (30, 40, 7), (22, 30, 7), (16, 20, 7),
          (22, 29, 3), (15, 20, 3)]
if len(sys.argv) > 1 and sys.argv[1] == 'child':
    import torch
    from gen6d_b200 import ops
    torch.manual_seed(0)
    for (H, W, k) in SHAPES:
        w = torch.rand(32, 512, k, k, device='cuda') * 0.05          # same-sign terms, like post-ReLU features
        pc = ops.pack_conv(w, None, pad=k // 2)
        x = torch.rand(1, H, W, 512, device='cuda')
        y = ops.conv(x, pc)
        os.environ['G6D_CONV_PATH'] = 'ffma'
        ref = ops.conv(x, pc)
        os.environ['G6D_CONV_PATH'] = 'tc'
        err = ((y - ref).abs().max() / ref.abs().max()).item()
        for _ in range(2): ops.conv(x, pc)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10): ops.conv(x, pc)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 2.0 * H * W * 32 * k * k * 512
        print(f'FLAT={os.environ.get("G6D_CONV_FLAT","1")} {H:3d}x{W:3d} k={k:2d} {ms*1e3:8.1f} us {fl/ms/1e9:6.1f} TF/s  rel err vs ffma {err:.2e}', flush=True)
else:
    for lvl in ('1', '2'):
        env = dict(os.environ, G6D_CONV_FLAT=lvl)
        subprocess.run([sys.executable, os.path.abspath(__file__), 'child'], env=env, check=False, timeout=280)
