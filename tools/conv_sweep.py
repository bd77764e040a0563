"""Time one conv shape across M for the tensor-core kernels (G6D_CONV_TC_V=1|2 chooses v1/v2)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gen6d_b200 import ops
os.environ['G6D_CONV_FLAT'] = '0'
cin, cout = 512, 512
w = torch.randn(cout, cin, 3, 3, device='cuda') * 0.02
pc = ops.pack_conv(w, torch.zeros(cout, device='cuda'), pad=1)
for (H, W) in ((22, 30), (40, 30), (60, 80), (60, 100), (88, 116), (120, 160)):
    x = torch.randn(1, H, W, cin, device='cuda')
    for _ in range(3): ops.conv(x, pc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): ops.conv(x, pc)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    M = H * W
    items = ((M + 127) // 128) * 4
    print(f'v{os.environ.get("G6D_CONV_TC_V","2")} M={M:6d} items={items:4d} {ms*1e3:8.1f} us  {2*M*cout*9*cin/ms/1e9:6.1f} TF/s')
