"""GroupNorm(+SiLU) device time on the UNet's batch-8 shapes (graph-timed), with a second, concatenated input where the UNet has a skip; the total weights each shape by how often the UNet runs it."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pfd_b200 import native as nv
from tools.gemm_perf import timeit

tot = 0.0
for (H, C1, C2, cnt) in [(64, 320, 0, 9), (64, 320, 320, 2), (64, 640, 320, 1), (32, 320, 0, 1), (32, 640, 0, 9), (32, 640, 640, 2),
                         (32, 1280, 640, 1), (32, 640, 320, 1), (16, 640, 0, 1), (16, 1280, 0, 9), (16, 1280, 1280, 2),
                         (16, 1280, 640, 1), (8, 1280, 0, 9), (8, 1280, 1280, 3)]:
    x1 = torch.randn(8, H, H, C1, device="cuda").half()
    x2 = torch.randn(8, H, H, C2, device="cuda").half() if C2 else None
    C = C1 + C2
    g, b = torch.randn(C, device="cuda").half(), torch.randn(C, device="cuda").half()
    out = torch.empty(8, H, H, C, device="cuda", dtype=torch.float16)

    def run():
        nv.gn_reset()
        nv.groupnorm(x1, g, b, 1e-5, silu=True, x2=x2, out=out)
    ms = timeit(run, n=10)
    tot += ms * cnt
    print(json.dumps(dict(H=H, C1=C1, C2=C2, us=round(ms * 1e3, 2), GBps=round(2 * 8 * H * H * C * 2 / ms / 1e6, 1))))
print(json.dumps(dict(total_ms_weighted=round(tot, 3))))
