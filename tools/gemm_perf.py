"""Per-shape throughput of the wgmma GEMM / implicit-GEMM conv kernel and the flash attention
kernel on the UNet's hot shapes (CUDA events, 3 warm-up + 10 timed launches, inputs >> L2 not enforced:
the same operands are reused, so these are L2-warm kernel rates; bench.py measures the cold-ish pipeline)."""
import json
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pfd_b200 import native as nv, attention as att

def timeit(fn, n=10):
    """Device time per launch: n launches captured in one CUDA graph (no host launch overhead)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

def main():
    dev = "cuda"
    res = []
    B = 8
    for (H, C, N) in [(64, 320, 320), (64, 640, 320), (64, 960, 320), (32, 640, 640), (32, 1280, 640), (32, 1920, 640),
                      (16, 1280, 1280), (16, 2560, 1280), (8, 1280, 1280), (8, 2560, 1280)]:
        x = torch.randn(B, H, H, C, device=dev).half()
        w = (torch.randn(N, 9 * C, device=dev) * (9 * C) ** -0.5).half()
        b = torch.randn(N, device=dev).half()
        out = torch.empty(B, H, H, N, device=dev, dtype=torch.float16)
        ms = timeit(lambda: nv.conv3x3(x, w, b, out=out))
        fl = 2.0 * B * H * H * N * 9 * C
        res.append(dict(op="conv3x3", B=B, HW=H, Cin=C, Cout=N, ms=ms, tflops=fl / ms / 1e9))
    for (M, N, K, act) in [(32768, 320, 320, 0), (32768, 2560, 320, 4), (32768, 320, 1280, 0), (8192, 640, 640, 0),
                           (8192, 5120, 640, 4), (8192, 640, 2560, 0), (2048, 1280, 1280, 0), (2048, 10240, 1280, 4),
                           (2048, 1280, 5120, 0), (8192, 8192, 8192, 0)]:
        x = torch.randn(M, K, device=dev).half()
        w = (torch.randn(N, K, device=dev) * K ** -0.5).half()
        bn = 0
        if act == 4:
            w, _, bn = nv.pack_geglu(w, None)
        out = torch.empty(M, N // 2 if act == 4 else N, device=dev, dtype=torch.float16)
        ms = timeit(lambda: nv.linear(x, w, None, act=act, out=out, bn_force=bn))
        res.append(dict(op="linear" + ("+geglu" if act == 4 else ""), M=M, N=N, K=K, ms=ms, tflops=2.0 * M * N * K / ms / 1e9))
    for (Bb, heads, Nq, Nk, d) in [(8, 8, 4096, 4096, 40), (8, 8, 4096, 148, 40), (8, 8, 1024, 1024, 80), (8, 8, 256, 256, 160)]:
        C = heads * d
        q = torch.randn(Bb * heads, Nq, d, device=dev).half()
        k = torch.zeros(Bb * heads, att.ceil8(Nk), d, device=dev).half(); k[:, :Nk] = torch.randn(Bb * heads, Nk, d, device=dev).half()
        vt = torch.zeros(Bb * heads, d, att.ceil8(Nk), device=dev).half(); vt[:, :, :Nk] = torch.randn(Bb * heads, d, Nk, device=dev).half()
        o = torch.empty(Bb, Nq, C, device=dev, dtype=torch.float16)
        for flash in (True, False):
            att.USE_FLASH = flash
            ms = timeit(lambda: att.attend(q, k, vt, B=Bb, heads=heads, Nq=Nq, Nk=Nk, scale=d ** -0.5, out=o), n=5)
            res.append(dict(op="attention" + ("_flash" if flash else "_unfused"), B=Bb, heads=heads, Nq=Nq, Nk=Nk, d=d, ms=ms,
                            tflops=4.0 * Bb * heads * Nq * Nk * d / ms / 1e9))
        att.USE_FLASH = True
    for r in res:
        print(json.dumps(r))

if __name__ == "__main__":
    main()
