"""Sweep the forced N-tile width for the Linear shapes of the UNet at batch 8 (one CFG pair of batch 4 at 512 x 512),
with the epilogue they run (bias_res = 1: bias + residual), including the swapped V^T products (weight as the A
operand).  Graph-timed device time in microseconds per launch; key "0" is the tile the library picks by itself."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pfd_b200 import native as nv
from tools.gemm_perf import timeit

dev = "cuda"
torch.manual_seed(0)
for (M, N, K, br) in [(32768, 320, 320, 1), (32768, 320, 1280, 1), (32768, 320, 320, 0), (32768, 640, 320, 0),
                      (8192, 640, 640, 1), (8192, 640, 2560, 1), (8192, 640, 640, 0), (8192, 1280, 640, 0),
                      (2048, 1280, 1280, 1), (2048, 1280, 5120, 1), (2048, 1280, 1280, 0), (2048, 2560, 1280, 0),
                      (512, 1280, 1280, 1), (1184, 1280, 768, 0), (1184, 320, 768, 0),
                      (320, 32768, 320, 0), (640, 8192, 640, 0), (1280, 2048, 1280, 0),
                      (32768, 960, 320, 0), (8192, 1920, 640, 0), (2048, 3840, 1280, 0)]:
    x = torch.randn(M, K, device=dev).half()
    w = (torch.randn(N, K, device=dev) * K ** -0.5).half()
    b = torch.randn(N, device=dev).half() if br else None
    r = torch.randn(M, N, device=dev).half() if br else None
    o = torch.empty(M, N, device=dev, dtype=torch.float16)
    row = dict(M=M, N=N, K=K, bias_res=br)
    for bn in (0, 64, 128, 160, 192, 256):
        try:
            row[bn] = round(timeit(lambda: nv.linear(x, w, b, residual=r, out=o, bn_force=bn), n=20) * 1e3, 1)
        except Exception as e:
            row[bn] = str(e)[:80]
    print(json.dumps(row))
