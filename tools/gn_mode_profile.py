"""GroupNorm device time per CFG-pair UNet evaluation (bench.py config 2: batch 4 -> 8 rows at 64x64 latents) in the
default and in the deterministic mode.  Each mode's evaluation is captured in a CUDA graph; torch.profiler sums the
device time of the GroupNorm kernels (and of the GEMMs, and of all kernels) over --reps replays.  The modes alternate
--rounds times in one process.  Run it with PFD_NO_PDL=1: with programmatic dependent launch a kernel starts before
its predecessor ends and waits, so its profiled duration includes that wait.

    PFD_NO_PDL=1 python tools/gn_mode_profile.py [--rounds 3] [--reps 10]
"""
import argparse
import json
import os
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import pfd_b200
    from pfd_b200 import get_model, model_cfg_bank
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    net = get_model()(model_cfg_bank()("pfd_seecoder"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    B, L = 4, 64
    g = torch.Generator().manual_seed(0)
    cond = (0.5 * torch.randn((B, 148, 768), generator=g)).cuda().half()
    c_full = torch.cat([torch.zeros_like(cond), cond])
    x = torch.randn((B, 4, L, L), generator=g).cuda().half()
    t_in = torch.full((2 * B,), 501, device="cuda", dtype=torch.long)
    prep = net.prepare_context(c_full, "image")
    c_info = {"type": "image", "c": prep["c"], "_pfd_prepared": prep, "control": None}

    def run():
        return net.apply_model({"type": "image", "x": torch.cat([x, x])}, t_in, c_info)

    res = {"device": torch.cuda.get_device_name(), "default": [], "deterministic": []}
    for _ in range(args.rounds):
        for mode in ("default", "deterministic"):
            pfd_b200.set_deterministic(mode == "deterministic")
            run()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                run()
            for _ in range(3):
                gr.replay()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    gr.replay()
                torch.cuda.synchronize()
            gn_us = gemm_us = total_us = 0.0
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                t = e.cuda_time_total if t is None else t
                total_us += t
                if "gn_" in e.key:
                    gn_us += t
                elif "gemm" in e.key:
                    gemm_us += t
            res[mode].append({"gn_ms": gn_us / args.reps / 1e3, "gemm_ms": gemm_us / args.reps / 1e3,
                              "kernels_ms": total_us / args.reps / 1e3})
            del gr
    pfd_b200.set_deterministic(False)
    for mode in ("default", "deterministic"):
        print(mode, " | ".join(f"gn {r['gn_ms']:.3f} gemm {r['gemm_ms']:.2f} all {r['kernels_ms']:.2f} ms" for r in res[mode]))
    print("GN_MODE_RESULT " + json.dumps(res))


if __name__ == "__main__":
    main()
