"""Fixed and per-K-block cost of one 128 x BN output tile of the GEMM kernel, per tile width and epilogue.

For every forced N-tile width BN and every epilogue the transformer Linears run, the product M = 32768, N = 5 * BN is
timed at K = 64 ... 2560 (1 to 40 K blocks of 64).  It has 1280 tiles, so the busiest CTA of a G-CTA grid runs
ceil(1280 / G) of them one after another, and

    device time / tiles per CTA  =  a + b * (K blocks)        (least squares over the K values)

a is what a tile costs besides its MMAs (epilogue, stores, pipeline refill), b is the time of one 128 x BN x 64 block.
One JSON line per (BN, epilogue): a and b in microseconds, the rms residual of the fit, and a in nanoseconds per
16-byte output chunk of the tile.  The first line names the card and its power limit (query only).

    python tools/gemm_tile_cost.py [--bn 64 128 ...] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

M = 32768
KS = (64, 320, 640, 1280, 2560)
WIDTHS = (64, 128, 160, 192, 256)
EPILOGUES = ("none", "bias", "bias_res", "geglu", "head_split")
HEAD_DIM = 40            # SD-1.5 self-attention at 64 x 64: 8 heads of 40; divides 5 * BN for every width


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return dict(card=name, power_limit=power, max_sm_clock=clock,
                sms=torch.cuda.get_device_properties(0).multi_processor_count)


def launcher(nv, ep, bn, K):
    N = 5 * bn
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
    b = None if ep == "none" else torch.randn(N, device="cuda").half()
    if ep == "geglu":           # the tile layout [value | gate] is a property of the weights' row order, not of the timing
        o = torch.empty(M, N // 2, device="cuda", dtype=torch.float16)
        return lambda: nv.linear(x, w, b, act=nv.ACT_GEGLU, out=o, bn_force=bn)
    if ep == "head_split":      # as attention.project_heads_fused: [B * T, heads * d] -> [B, heads, T, d]
        B, T, d = 8, M // 8, HEAD_DIM
        vh = N // d
        o = torch.empty((B, vh, T, d), device="cuda", dtype=torch.float16)
        return lambda: nv.gemm_raw([(x, 1, K, (K, K * T, K * T))], in_w=T, in_h=1, stride=1, W=T, H=1, NB=B, w=w, N=N,
                                   K=K, bias=b, out=o, so=(vh * T * d, 0, 0, d, T * d, 1), ndiv=1, cdiv=d, bn_force=bn)
    r = torch.randn(M, N, device="cuda").half() if ep == "bias_res" else None
    o = torch.empty(M, N, device="cuda", dtype=torch.float16)
    return lambda: nv.linear(x, w, b, residual=r, out=o, bn_force=bn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bn", type=int, nargs="+", default=list(WIDTHS))
    ap.add_argument("--epilogue", nargs="+", default=list(EPILOGUES), choices=EPILOGUES)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_tile_cost.py needs a CUDA device")
    from pfd_b200 import native as nv
    from tools.gemm_perf import timeit
    info = card()
    print(json.dumps(info), flush=True)
    tiles_per_cta = -(-(M // 128) * 5 // info["sms"])
    torch.manual_seed(0)
    for bn in args.bn:
        for ep in args.epilogue:
            us = [timeit(launcher(nv, ep, bn, K), n=args.reps) * 1e3 / tiles_per_cta for K in KS]
            kb = np.array([K // 64 for K in KS], dtype=np.float64)
            A = np.stack([np.ones_like(kb), kb], axis=1)
            (a, b), *_ = np.linalg.lstsq(A, np.array(us), rcond=None)
            rms = float(np.sqrt(np.mean((A @ np.array([a, b]) - us) ** 2)))
            chunks = 128 * (bn // 2 if ep == "geglu" else bn) // 8
            print(json.dumps(dict(bn=bn, epilogue=ep, a_us=round(float(a), 3), b_us=round(float(b), 4),
                                  fit_rms_us=round(rms, 3), a_ns_per_chunk=round(float(a) * 1e3 / chunks, 2),
                                  us_per_tile={str(K): round(u, 2) for K, u in zip(KS, us)})), flush=True)


if __name__ == "__main__":
    main()
