"""Time seeded (per-sample, on-device noise) against unseeded stochastic sampling at the size of bench.py's config 2
(64x64 latents, batch 4, CFG scale 2, synthetic weights), and the noise kernel alone:
  - DDIM-50 eta 0 (one graph for the whole loop), the per-step cost a seeded stochastic loop is compared with;
  - DDIM-50 eta 1: unseeded (one-step graph + host noise per step) vs seeded (one graph for the whole loop);
  - euler_a-50 eta 1: unseeded (one-step graph + host noise per step) vs seeded (one graph);
  - dpmpp_2m_sde at 20 and 25 steps, eta 1, unseeded vs seeded;
  - pfd_randn_f16 at [4, 4, 64, 64] (CUDA events around a graph of 200 back-to-back launches).
Reported per run: ms per sample() call (the denoising loop only), ms per step, latents per second.  The card's name and
power limit are read in the same run.

    python tools/rng_perf.py [--iters 3] [--out results/rng_perf.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.sampler_perf import B, GUIDANCE, LAT, timed  # noqa: E402

RUNS = [("ddim", 50, 0.0, (False,))] + [(k, n, 1.0, (False, True)) for k, n in
                                          (("ddim", 50), ("euler_a", 50), ("dpmpp_2m_sde", 20), ("dpmpp_2m_sde", 25))]


def randn_kernel_us(n_launch=200):
    from pfd_b200 import native as nv
    from pfd_b200.rng import seeds_tensor
    import numpy as np
    out = torch.empty((B, 4, LAT, LAT), device="cuda", dtype=torch.float16)
    seeds = seeds_tensor(np.arange(B, dtype=np.uint64), "cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    launch = lambda: nv.randn_f16(out, seeds, 1, 0, step)
    launch()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(n_launch):
            launch()
    return 1e3 * timed(graph.replay, 5, warmup=2) / n_launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from pfd_b200 import DDIMSampler, Sampler, get_model, model_cfg_bank
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"[rng-perf] {gpu}")
    net = get_model()(model_cfg_bank()("pfd_seecoder"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    net.eval()
    g = torch.Generator().manual_seed(0)
    cond = (0.5 * torch.randn((B, 148, 768), generator=g)).half().cuda()
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": GUIDANCE, "control": None}
    shape = [B, 4, LAT, LAT]
    rows = []
    for kind, steps, eta, variants in RUNS:
        for seeded in variants:
            smp = DDIMSampler(net) if kind == "ddim" else Sampler(net, type=kind)

            def fn():
                x_info = {"type": "image"}
                if seeded:
                    x_info["seeds"] = 1000
                if kind == "ddim":
                    smp.sample(steps=steps, shape=shape, x_info=x_info, c_info=dict(c_info), verbose=False, eta=eta)
                else:
                    smp.sample(steps=steps, shape=shape, x_info=x_info, c_info=dict(c_info), eta=eta)
            ms = timed(fn, args.iters)
            row = {"sampler": kind, "steps": steps, "eta": eta, "seeded": seeded, "ms_per_call": round(ms, 1),
                   "ms_per_step": round(ms / steps, 2), "latents_per_s": round(B * 1e3 / ms, 3)}
            print(f"[rng-perf] {json.dumps(row)}")
            rows.append(row)
            del smp
            torch.cuda.empty_cache()
    us = randn_kernel_us()
    print(f"[rng-perf] pfd_randn_f16 at [{B},4,{LAT},{LAT}]: {us:.2f} us per launch")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "batch": B, "latent": LAT, "guidance": GUIDANCE, "rows": rows,
                       "randn_kernel_us": round(us, 2)}, f, indent=1)


if __name__ == "__main__":
    main()
