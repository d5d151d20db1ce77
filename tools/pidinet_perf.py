"""Time the PiDiNet annotator on the GPU with CUDA events (synthetic weights; the time does not depend on the weight
values), at 512^2 .. 1536^2 and batch 1 / 4: pidinet.preprocess_pidinet and the whole
ControlNet.preprocess(type='scribble') (PiDiNet + make_scribble).  When the reference is staged under oracle/_ref,
also time its pidinet() network in fp32 eager on the same GPU (network only: apply_pidinet's numpy post-processing
runs on the CPU and is not timed), for the same images one at a time, as apply_pidinet does.  Prints the card name
and power limit read in the same run.

    python tools/pidinet_perf.py [--iters 20] [--out results/pidinet_perf.json]
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
    """Multiply-adds x 2 of every conv at H x W -> (total, CDCM dilated convs)."""
    from oracle.pidinet_oracle import DIL, STAGE_CH, block_names
    f = 2 * H * W * 27 * STAGE_CH[0]                                    # init block
    for _, s, layer, cin, cout, stride in block_names():
        h, w = H >> s, W >> s
        ks = 25 if layer % 4 == 2 else 9
        f += 2 * h * w * (cin * ks + cin * cout + (cin * cout if stride > 1 else 0))
    dil = 0
    for s in range(4):
        h, w = H >> s, W >> s
        f += 2 * h * w * (STAGE_CH[s] * DIL + 4 * DIL + 36 + DIL)        # CDCM 1x1, CSAM, MapReduce
        dil += 2 * h * w * 4 * 9 * DIL * DIL
    return (f + dil) / 1e9, dil / 1e9


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
    from oracle.pidinet_oracle import fill_synthetic
    from pfd_b200 import pidinet
    from pfd_b200.scribble import preprocess_scribble
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"[pidinet-perf] {gpu}")
    net = fill_synthetic(pidinet.PiDiNet().cuda(), seed=0)
    pidinet.set_network(net)
    ref = None
    from tools import ref_harness
    if ref_harness.available():
        cwd = os.getcwd()
        ref_harness.import_reference()
        import lib.model_zoo.controlnet_annotator.pidinet as refpidi
        os.chdir(cwd)
        ref = fill_synthetic(refpidi.pidinet(), seed=0).cuda().float().eval()
    rows = []
    for S in SIZES:
        for B in BATCHES:
            x = torch.rand((B, 3, S, S), device="cuda", dtype=torch.float16)
            total, dil = gflop(S, S)
            ms = timed(lambda: pidinet.preprocess_pidinet(x), args.iters)
            ms_scr = timed(lambda: preprocess_scribble(x), args.iters)
            row = {"size": S, "batch": B, "pidinet_ms": round(ms, 3), "scribble_ms": round(ms_scr, 3),
                   "gflop": round(B * total, 1), "cdcm_gflop": round(B * dil, 1), "tflops": round(B * total / ms, 1)}
            if ref is not None:
                xr = x.float().mul(255).floor().flip(1) / 255.0
                with torch.no_grad():
                    row["ref_fp32_ms"] = round(timed(lambda: [ref(xr[b:b + 1]) for b in range(B)],
                                                     max(3, args.iters // 4), warmup=2), 3)
            print(f"[pidinet-perf] {json.dumps(row)}")
            rows.append(row)
            del x
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
