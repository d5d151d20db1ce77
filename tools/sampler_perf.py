"""Time the samplers at the size of bench.py's config 2 (512x512 output = 64x64 latents, batch 4, CFG scale 2, i.e. a
CFG batch of 8 per UNet evaluation) with synthetic weights: DDIM-50 (eta 0: one graph for the whole loop), euler_a-50
(eta 1: one graph replay plus one host noise draw per step, as DDIM with eta > 0 and no seeds runs), euler_a-50 with
eta 0 and dpmpp_2m-20 / 25 (one graph for the whole loop).  Reported per
sampler: ms per sample() call (the denoising loop only: no SeeCoder, no VAE), ms per step, latents per second, and
the k-sampler update kernel's own time (CUDA events around a graph of 200 back-to-back launches).  The card's name and
power limit are read in the same run.

    python tools/sampler_perf.py [--iters 3] [--out results/sampler_perf.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, LAT, GUIDANCE = 4, 64, 2.0
RUNS = [("ddim", 50, 0.0), ("euler_a", 50, 1.0), ("euler_a", 50, 0.0), ("dpmpp_2m", 20, 0.0), ("dpmpp_2m", 25, 0.0)]


def timed(fn, iters, warmup=1):
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


def update_kernel_us(n_launch=200):
    from pfd_b200 import native as nv
    shape = (B, 4, LAT, LAT)
    eps = torch.randn((2 * B,) + shape[1:], device="cuda").half()
    x = torch.randn(shape, device="cuda")
    d = torch.zeros_like(x)
    xin = torch.empty_like(eps)
    out = torch.empty(shape, device="cuda", dtype=torch.float16)
    noise = torch.randn(shape, device="cuda").half()
    coef = torch.tensor([[1.0, 0.9, 0.1, 0.0, 0.05, 0.5]] * 2, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    launch = lambda: nv.ksampler_step(eps, True, GUIDANCE, coef, step, 1, x, d, xin, out, noise=noise)
    launch()
    torch.cuda.synchronize()
    # the launches are captured into a graph, as in the sampler, so the host's ctypes call cost is not timed
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
    print(f"[sampler-perf] {gpu}")
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
    for kind, steps, eta in RUNS:
        if kind == "ddim":
            smp = DDIMSampler(net)
            fn = lambda: smp.sample(steps=steps, shape=shape, x_info={"type": "image"}, c_info=dict(c_info),
                                    verbose=False, eta=eta)
        else:
            smp = Sampler(net, type=kind)
            fn = lambda: smp.sample(steps=steps, shape=shape, x_info={"type": "image"}, c_info=dict(c_info), eta=eta)
        ms = timed(fn, args.iters)
        row = {"sampler": kind, "steps": steps, "eta": eta, "ms_per_call": round(ms, 1),
               "ms_per_step": round(ms / steps, 2), "latents_per_s": round(B * 1e3 / ms, 3)}
        print(f"[sampler-perf] {json.dumps(row)}")
        rows.append(row)
        del smp
        torch.cuda.empty_cache()
    us = update_kernel_us()
    print(f"[sampler-perf] pfd_ksampler_step_f32 at [{B},4,{LAT},{LAT}] with CFG and noise: {us:.2f} us per launch")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "batch": B, "latent": LAT, "guidance": GUIDANCE, "rows": rows,
                       "update_kernel_us": round(us, 2)}, f, indent=1)


if __name__ == "__main__":
    main()
