"""Micro-benchmark of the tensor-core (wgmma) Linear (dev tool): CUDA-event time per call for the GEMM shapes of the 3DMatch model.
Run from any checkout: uses the package next to this file's parent directory (or GEOB_ROOT)."""
import os
import sys

ROOT = os.environ.get('GEOB_ROOT', os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch

from geotransformer_b200 import functional as GF

SHAPES = [(40000, 64, 32), (40000, 480, 32), (40000, 32, 128), (40000, 64, 128), (12000, 960, 64), (12000, 64, 256), (3400, 1920, 128),
          (3400, 128, 512), (640, 3840, 256), (640, 256, 1024), (640, 1024, 256), (640, 256, 768), (320, 256, 256), (640, 256, 512)]
print('root', ROOT)
if os.environ.get('GEOB200_LINEAR_PERSISTENT'):
    from geotransformer_b200 import _lib
    _lib.lib().geob200_set_linear_persistent(1)
    print('persistent tile loop ON')
for m, k, n in SHAPES:
    x = torch.randn(m, k, device='cuda')
    w = torch.randn(n, k, device='cuda')
    b = torch.randn(n, device='cuda')
    out = torch.empty(m, n, device='cuda')
    for _ in range(5):
        GF.linear(x, w, b, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        GF.linear(x, w, b, out=out)
    e1.record()
    torch.cuda.synchronize()
    print(f'{m:6d} x {k:5d} -> {n:5d}: {e0.elapsed_time(e1) / 50 * 1e3:8.1f} us')
