"""Time ControlNet.preprocess(type='scribble') on the GPU with CUDA events, for method='hed' (HED network plus the
make_scribble kernels; synthetic HED weights, the time does not depend on their values) and method='xdog', at 512^2 ..
1536^2 and batch 1 / 4, plus the post-process kernels alone (pfd_scribble_hed_f32 on a ready HED map, and
pfd_scribble_xdog_f32, which is the whole xdog path).  When cv2 is importable it also times, on the host cores, what the
reference runs there per image: the cv2 calls of make_scribble (controlnet.py:436-454) and of the xdog lines
(controlnet.py:476-482).  The card's name, power limit and maximum SM clock are printed in the same run.

    python tools/scribble_perf.py [--iters 20] [--out results/scribble_perf.json]
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


def host_ms(fn, iters):
    fn()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t) * 1e3 / iters


def cv2_tails():
    """The reference's host-side cv2 work of make_scribble and xdog on one image, or None without cv2."""
    try:
        import cv2
    except ImportError:
        return None
    lines = [np.array(a, np.uint8) for a in ([[0, 0, 0], [1, 1, 1], [0, 0, 0]], [[0, 1, 0], [0, 1, 0], [0, 1, 0]],
                                             [[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[0, 0, 1], [0, 1, 0], [1, 0, 0]])]

    def make_scribble(r):
        x = cv2.GaussianBlur(r.astype(np.float32), (0, 0), 3.0)
        y = np.zeros_like(x)
        for f in lines:
            np.putmask(y, cv2.dilate(x, kernel=f) == x, x)
        z = np.zeros_like(y, dtype=np.uint8)
        z[y > 127] = 255
        r = cv2.GaussianBlur(z, (0, 0), 3.0)
        r[r > 4] = 255
        r[r < 255] = 0
        return r

    def xdog(img, threshold=32):
        g1 = cv2.GaussianBlur(img.astype(np.float32), (0, 0), 0.5)
        g2 = cv2.GaussianBlur(img.astype(np.float32), (0, 0), 5.0)
        dog = (255 - np.min(g2 - g1, axis=2)).clip(0, 255).astype(np.uint8)
        result = np.zeros_like(img, dtype=np.uint8)
        result[2 * (255 - dog) > threshold] = 255
        return result

    return make_scribble, xdog, cv2.getNumThreads()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle.hed_oracle import fill_synthetic, hed_image
    from pfd_b200 import hed, native as nv
    from pfd_b200.controlnet import ControlNet
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"[scribble-perf] {gpu}")
    hed.set_network(fill_synthetic(hed.ControlNetHED().cuda(), seed=0))
    ctl = ControlNet(32, 4, 32, 3, 1, [], channel_mult=(1,), use_spatial_transformer=True, context_dim=32,
                     num_heads=1, legacy=False).cuda()
    tails = cv2_tails()
    print(f"[scribble-perf] host tail: {'cv2 with %d threads' % tails[2] if tails else 'cv2 not importable'}, "
          f"{os.cpu_count()} host cores")
    rows = []
    for S in SIZES:
        img = hed_image(S, S, S)
        for B in BATCHES:
            x = (torch.from_numpy(img).permute(2, 0, 1)[None].float() / 255).repeat(B, 1, 1, 1).cuda().half()
            row = {"size": S, "batch": B}
            row["hed_ms"] = timed(lambda: ctl.preprocess(x, type="scribble", method="hed"), args.iters)
            row["xdog_ms"] = timed(lambda: ctl.preprocess(x, type="scribble", method="xdog"), args.iters)
            hmap = hed.preprocess_hed(x)
            row["hed_post_kernels_ms"] = timed(lambda: nv.scribble_hed(hmap), args.iters)
            row["xdog_kernel_ms"] = timed(lambda: nv.scribble_xdog(x, 32), args.iters)
            if tails is not None and B == 1:
                make_scribble, xdog, _ = tails
                lv = (hmap[0, 0].double() * 255).round().to(torch.uint8).cpu().numpy()
                it = max(2, args.iters // 4)
                row["cv2_make_scribble_ms_per_image"] = host_ms(lambda: make_scribble(lv), it)
                row["cv2_xdog_ms_per_image"] = host_ms(lambda: xdog(img), it)
            row = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in row.items()}
            print(f"[scribble-perf] {json.dumps(row)}")
            rows.append(row)
            del x, hmap
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
