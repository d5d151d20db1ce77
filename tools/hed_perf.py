"""Time ControlNet.preprocess(type='hed') on the GPU with CUDA events (synthetic weights; the time does not depend on
the weight values), at 512^2 .. 1536^2 and batch 1 / 4.  When the reference is staged under oracle/_ref, also time its
ControlNetHED_Apache2 network in fp32 eager on the same GPU (network only: apply_hed's resize / sigmoid run on the CPU
and are not timed), for the same images one at a time, as apply_hed does.

    python tools/hed_perf.py [--iters 20] [--out results/hed_perf.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [512, 768, 1024, 1536]
BATCHES = [1, 4]


def gflop(H, W):
    """Multiply-adds x 2 of the 13 convolutions and 5 projections at H x W."""
    from oracle.hed_oracle import BLOCKS
    f, h, w = 0, H, W
    for bi, (cin, cout, layers) in enumerate(BLOCKS):
        if bi:
            h, w = h // 2, w // 2
        for li in range(layers):
            f += 2 * h * w * 9 * (cin if li == 0 else cout) * cout
        f += 2 * h * w * cout
    return f / 1e9


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle.hed_oracle import fill_synthetic
    from pfd_b200 import hed
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"[hed-perf] {gpu}")
    net = fill_synthetic(hed.ControlNetHED().cuda(), seed=0)
    hed.set_network(net)
    ref = None
    from tools import ref_harness
    if ref_harness.available():
        cwd = os.getcwd()
        ref_harness.import_reference()
        import lib.model_zoo.controlnet_annotator.hed as refhed
        os.chdir(cwd)
        ref = fill_synthetic(refhed.ControlNetHED_Apache2(), seed=0).cuda().float().eval()
    rows = []
    for S in SIZES:
        for B in BATCHES:
            x = torch.rand((B, 3, S, S), device="cuda", dtype=torch.float16)
            ms = timed(lambda: hed.preprocess_hed(x), args.iters)
            row = {"size": S, "batch": B, "ms": round(ms, 3), "gflop": round(B * gflop(S, S), 1),
                   "tflops": round(B * gflop(S, S) / ms, 1)}
            if ref is not None:
                xr = (x.float() * 255).floor()
                with torch.no_grad():
                    row["ref_fp32_ms"] = round(timed(lambda: [ref(xr[b:b + 1]) for b in range(B)],
                                                     max(3, args.iters // 4), warmup=2), 3)
            print(f"[hed-perf] {json.dumps(row)}")
            rows.append(row)
            del x
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
