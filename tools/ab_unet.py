"""A/B timing of one CFG-pair UNet evaluation (BASELINE configs[1]: batch 4 -> 8 samples at 64x64) under several library
settings INSIDE ONE PROCESS, interleaved, so that box-to-box spread and the power/thermal state do not bias the
comparison (r2: three separate bench.py runs on one box disagreed by 4 % in the opposite direction of their own
per-kernel breakdowns).  Each variant is captured into its own CUDA graph; rounds alternate between the graphs.

    python tools/ab_unet.py [--rounds 6] [--reps 20] [--control] [--env-variant name=option:value ...]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--control", action="store_true")
    ap.add_argument("--env-variant", action="append", default=[],
                    help="name=OPTION:value - an extra variant that sets a library option (pfd_set_option) before capture")
    args = ap.parse_args()
    from pfd_b200 import get_model, model_cfg_bank, native as nv
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet" if args.control else "pfd_seecoder"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    B, L = args.batch, args.res // 8
    g = torch.Generator().manual_seed(0)
    cond = (0.5 * torch.randn((B, 148, 768), generator=g)).cuda().half()
    c_full = torch.cat([torch.zeros_like(cond), cond])
    x = torch.randn((B, 4, L, L), generator=g).cuda().half()
    t_in = torch.full((2 * B,), 501, device="cuda", dtype=torch.long)
    hint = (torch.rand((1, 3, args.res, args.res), generator=g) > 0.9).half().cuda() if args.control else None
    prep = net.prepare_context(c_full, "image")
    if hint is not None:
        prep["hint"] = net.ctl.hint_features(hint)
    c_info = {"type": "image", "c": prep["c"], "_pfd_prepared": prep, "control": hint}

    def run():
        return net.apply_model({"type": "image", "x": torch.cat([x, x])}, t_in, c_info)

    # name -> callable applied before that variant's warm-up + capture (library switches, python-level toggles ...)
    variants = {"default": lambda: None}
    for spec in args.env_variant:                      # e.g. --env-variant det=deterministic:1
        vname, kv = spec.split("=", 1)
        key, val = kv.split(":", 1)
        variants[vname] = (lambda k=key, v=val: nv.set_env_option(k, v))
    graphs = {}
    for name, setup in variants.items():
        nv.set_env_option(None, None)                  # back to the defaults
        setup()
        run()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            out = run()
        graphs[name] = (gr, out)
    nv.set_env_option(None, None)
    ref = None
    times = {k: [] for k in graphs}
    for gr, _ in graphs.values():
        for _ in range(5):
            gr.replay()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for name, (gr, out) in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.reps)
    res = {}
    for name, (gr, out) in graphs.items():
        ts = sorted(times[name])
        o = out.float()
        if ref is None:
            ref = o
        res[name] = {"ms_median": ts[len(ts) // 2], "ms_min": ts[0], "ms_max": ts[-1],
                     "rel_rms_vs_first": ((o - ref).pow(2).mean() / ref.pow(2).mean()).sqrt().item()}
        print(f"{name:45s} median {ts[len(ts) // 2]:.3f} ms  (min {ts[0]:.3f}, max {ts[-1]:.3f})  rel vs first {res[name]['rel_rms_vs_first']:.2e}")
    print("AB_RESULT " + json.dumps(res))


if __name__ == "__main__":
    main()
