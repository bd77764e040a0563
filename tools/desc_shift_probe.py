"""Checks that a row-shifted K-major SWIZZLE_128B wgmma descriptor reads what the flat convolution kernel wrote
(rows listed as bad disagree with the expected product)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gen6d_b200 import _lib
lib = _lib.lib()
torch.set_printoptions(linewidth=200, precision=4)
for mode, shift in ((0, 0), (0, 3), (1, 3)):
    out = torch.zeros(64, 32, device='cuda')
    lib.g6d_debug_desc_shift(ctypes.c_void_p(out.data_ptr()), shift, mode, None)
    torch.cuda.synchronize()
    got = out.cpu()
    r = torch.arange(64, dtype=torch.float32)[:, None] + shift
    want = r + torch.arange(32, dtype=torch.float32)[None] / 64
    want = (want.view(torch.int32) & ~0x1FFF).view(torch.float32)   # the tf32 MMA ignores the low 13 bits of A
    bad = (got - want).abs().max(1)[0].ge(1e-3).nonzero().flatten().tolist()
    print('mode', mode, 'shift', shift, 'bad rows', bad[:40], '...' if len(bad) > 40 else '')
    for rr in bad[:3] + bad[-2:]:
        print('  row', rr, 'got', got[rr, :8].tolist(), '| col 8..', got[rr, 8:12].tolist(), 'want', want[rr, :2].tolist())
