"""Time the M-LSD annotator on the GPU with CUDA events (synthetic weights; the time does not depend on the weight
values beyond the number of segments drawn), at 512^2 .. 1536^2 and batch 1 / 4: the whole
ControlNet.preprocess(type='mlsd') path, pfd_b200.mlsd.preprocess_mlsd.  TFLOP/s counts the network's convolutions
from their shapes.  When the reference is staged under oracle/_ref, also time its MobileV2_MLSD_Large in fp32 eager on
the same GPU, one image at a time as apply_mlsd runs it, and separately its host-side decode and drawing
(deccode_output_score_and_ptss from the network output, the segment loop and cv2.line, per image).  Prints the card
name and power limit read in the same run.

    python tools/mlsd_perf.py [--iters 20] [--out results/mlsd_perf.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [512, 768, 1024, 1536]
BATCHES = [1, 4]


def gflop(H, W):
    """2 x multiply-adds of every conv of the network on one H x W image (channels 7..11 of the last 1x1 only)."""
    from oracle.mlsd_oracle import DECODER, trunk_layers
    h, w = H // 2, W // 2
    f = 2 * h * w * 9 * 4 * 32                                               # stem
    sizes = {0: (h, w)}
    cur = (h, w)
    for i, inp, hid, oup, stride, _ in trunk_layers():
        hi, wi = cur
        cur = (hi // stride, wi // stride)
        ho, wo = cur
        f += 2 * hi * wi * inp * hid * (hid != inp) + 2 * ho * wo * (9 * hid + hid * oup)
        sizes[i] = cur
    res = [sizes[13], sizes[6], sizes[3], sizes[1]]
    for k, (_, c1, c2, up) in enumerate(DECODER):
        ha, wa = res[k]
        hb, wb = (ha // 2, wa // 2) if up else (ha, wa)
        f += 2 * ha * wa * c1 * 64 + 2 * hb * wb * c2 * 64
        f += 2 * ha * wa * 9 * 128 * (128 + 64)
    f += 2 * h * w * 9 * 64 * 64 * 2 + 2 * h * w * 64 * 5                   # block23
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
    from oracle.mlsd_oracle import fill_synthetic
    from pfd_b200 import mlsd
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"[mlsd-perf] {gpu}")
    net = fill_synthetic(mlsd.MLSD().cuda(), seed=0)
    mlsd.set_network(net)
    ref = refutils = None
    from tools import ref_harness
    if ref_harness.available():
        cwd = os.getcwd()
        ref_harness.import_reference()
        from lib.model_zoo.controlnet_annotator.mlsd import utils as refutils
        from lib.model_zoo.controlnet_annotator.mlsd.models.mbv2_mlsd_large import MobileV2_MLSD_Large
        os.chdir(cwd)
        ref = fill_synthetic(MobileV2_MLSD_Large(), seed=0).cuda().float().eval()
    import cv2
    warm = torch.rand((1, 3, SIZES[0], SIZES[0]), device="cuda", dtype=torch.float16)
    timed(lambda: mlsd.preprocess_mlsd(warm), args.iters)            # first launches and clocks out of the table
    rows = []
    for S in SIZES:
        for B in BATCHES:
            x = torch.rand((B, 3, S, S), device="cuda", dtype=torch.float16)
            g = gflop(S, S) * B
            ms = timed(lambda: mlsd.preprocess_mlsd(x), args.iters)
            row = {"size": S, "batch": B, "mlsd_ms": round(ms, 3), "gflop": round(g, 1), "tflops": round(g / ms, 1)}
            if ref is not None:
                xr = torch.cat([x.float().mul(255).floor(), torch.ones((B, 1, S, S), device="cuda")], 1) / 127.5 - 1
                with torch.no_grad():
                    row["ref_fp32_ms"] = round(timed(lambda: [ref(xr[b:b + 1]) for b in range(B)],
                                                     max(3, args.iters // 4), warmup=2), 3)
                    outs = [ref(xr[b:b + 1]).cpu() for b in range(B)]

                def host_post():
                    for o in outs:
                        pts, scores, vmap = refutils.deccode_output_score_and_ptss(o, 200, 3)
                        canvas = np.zeros((S, S, 3), np.uint8)
                        for (y, xx), s in zip(pts, scores):
                            d = vmap[y, xx]
                            if s > 0.1 and np.sqrt(np.sum((d[:2] - d[2:]) ** 2)) > 0.1:
                                p = [int(2 * (v + c)) for v, c in zip(d, (xx, y, xx, y))]
                                cv2.line(canvas, (p[0], p[1]), (p[2], p[3]), [255, 255, 255], 1)
                host_post()
                t = time.perf_counter()
                for _ in range(3):
                    host_post()
                row["ref_host_post_ms"] = round((time.perf_counter() - t) / 3 * 1e3, 3)
            print(f"[mlsd-perf] {json.dumps(row)}")
            rows.append(row)
            del x
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
