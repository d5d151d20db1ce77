"""Is the wgmma GEMM main loop limited by operand feed from L2?

For the UNet's long-K 3x3 convolutions and its K = 320 / 1280 linears (batch 8 = one CFG pair of batch 4 at 512 x 512)
the kernel is timed with every N tile width (bn_force).  Every 64-wide K block of a 128 x BN tile reads 16 KiB of A and
BN * 128 B of B for 2 * 128 * BN * 64 FLOP, so a wider tile needs fewer operand bytes per FLOP (kib_per_mflop).  If the
rate climbs with that intensity at a similar wave count, the main loop is feed-bound.  `tflops` counts the problem's
FLOPs; `tile_tflops` counts every computed tile including the N padding (N not a multiple of BN), which is the fair
per-tile comparison between widths.  torch.matmul (cuBLAS) on the same M x N x K (for the convs: the im2col'ed
problem, gather not included) is printed as a yardstick for what the card reaches.  Times are CUDA-event timed graph
replays (tools/gemm_perf.py), so operands are L2-warm.

    python tools/gemm_feed_probe.py [--reps 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pfd_b200 import native as nv
from tools.gemm_perf import timeit

BM, BK = 128, 64


def kib_per_mflop(bn):
    return (BM * BK * 2 + bn * BK * 2) / 1024.0 / (2.0 * BM * bn * BK / 1e6)


def conv_call(B, H, C, N):
    x = torch.randn(B, H, H, C, device="cuda").half()
    w = (torch.randn(N, 9 * C, device="cuda") * (9 * C) ** -0.5).half()
    b = torch.randn(N, device="cuda").half()
    out = torch.empty(B, H, H, N, device="cuda", dtype=torch.float16)

    def run(bn):
        nv.gemm_raw([(x, 9, C, (x.stride(2), x.stride(1), x.stride(0)))], in_w=H, in_h=H, stride=1, W=H, H=H, NB=B,
                    w=w, N=N, K=w.stride(0), bias=b, out=out, so=(out.stride(0), 0, out.stride(1), out.stride(2), 0, 1),
                    bn_force=bn)
    a2 = x.reshape(B * H * H, C).repeat(1, 9)
    # every 128-row tile holds 128 output pixels of the raster (64 x 2, 32 x 4 or 16 x 8 pixels: no row padding)
    return run, B * H * H, N, 9 * C, (lambda: torch.matmul(a2, w.t()))


def linear_call(M, N, K):
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
    out = torch.empty(M, N, device="cuda", dtype=torch.float16)
    return (lambda bn: nv.linear(x, w, None, out=out, bn_force=bn)), M, N, K, (lambda: torch.matmul(x, w.t()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.manual_seed(0)
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    print(f"# {props.name}, {sms} SMs")
    shapes = [("conv3x3 320->320 @64 NB=8", conv_call, (8, 64, 320, 320)),
              ("conv3x3 640->640 @32 NB=8", conv_call, (8, 32, 640, 640)),
              ("conv3x3 1280->1280 @16 NB=8", conv_call, (8, 16, 1280, 1280)),
              ("linear M=32768 N=320 K=320", linear_call, (32768, 320, 320)),
              ("linear M=32768 N=320 K=1280", linear_call, (32768, 320, 1280))]
    for name, mk, shp in shapes:
        run, M, N, K, ref = mk(*shp)
        flops = 2.0 * M * N * K
        ms = timeit(ref, n=args.reps)
        print(json.dumps({"shape": name, "impl": "torch.matmul", "ms": round(ms, 4),
                          "tflops": round(flops / ms / 1e9, 1)}))
        for bn in (64, 128, 160, 256):
            ms = timeit(lambda: run(bn), n=args.reps)
            m_t, n_t = -(-M // BM), -(-N // bn)
            tile_flops = 2.0 * m_t * BM * n_t * bn * K
            print(json.dumps({"shape": name, "impl": "pfd", "bn": bn, "ms": round(ms, 4),
                              "tflops": round(flops / ms / 1e9, 1), "tile_tflops": round(tile_flops / ms / 1e9, 1),
                              "tiles": m_t * n_t, "waves": round(m_t * n_t / sms, 2),
                              "kib_per_mflop": round(kib_per_mflop(bn), 2)}))


if __name__ == "__main__":
    main()
