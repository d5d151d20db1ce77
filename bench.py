#!/usr/bin/env python
"""Benchmark of the Prompt-Free-Diffusion hot path on an H100.

  python bench.py --gpus N --steps K --warmup W [--config C] [--dump-outputs DIR]   # our CUDA path (pfd_b200)
  python bench.py --impl reference --gpus N --steps K ...      # the reference's own CPU path on the host cores
                                                               # (unmodified reference modules from oracle/_ref;
                                                               #  oracle port when the staged copy is absent)

Workloads = BASELINE.json configs (SURVEY.md §8d), per GPU; --config 2 (the one the metric is quoted on) is the
default: 512x512, SeeCoder + SD-v1.5 UNet, 50 DDIM steps, CFG 2.0, batch 4, fp16, synthetic seeded weights/inputs.
  1: 256x256 reference image, 10 steps, batch 1, 512x512 output      3: config 2 with batch 8 and the zero-padded
  4: config 2 + ControlNet (512x512 binary hint), batch 4 per GPU       [77,768] "anime" unconditional context
  5: 768x768, steps=30 (31 evaluations), SeeCoder-PA (PPE_MLP), batch 4 per GPU
One "step" = one full request (SeeCoder encode of one reference image -> all DDIM steps for the batch -> AutoKL
decode).  Multi-GPU = pure batch split: by default every rank serves its own request (weak scaling, no data-path
collective; NCCL only for the barrier / max-over-ranks timing); --split shards ONE request of `batch` images over the
ranks with pfd_b200/parallel.py (rank-0 encode + broadcast, full-batch randn + slice, all-gather of the images).

The default run also times, on rank 0 at N = 1: `gpu_reference` = the UNMODIFIED reference modules in PyTorch eager
fp16 on the same GPU and the same request (the north-star's x2 denominator; reported as `vs_baseline`), and
`cpu_baseline` = the reference's CPU path on the host cores on a bounded sample.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

METRIC = "512x512 images/sec @ 50 DDIM steps"
# per-image algorithmic TFLOP (SURVEY.md §8d): evals * (UNet [+ControlNet]) + VAE + SeeCoder / B
CONFIGS = {
    1: dict(res=512, ref_res=256, ddim_steps=10, batch=1, control=False, pa=False, anime=False, f_img=18.92,
            name="configs[0] geometry on the GPU: 256x256 ref image, 10 DDIM steps, batch 1, 512x512 output"),
    2: dict(res=512, ref_res=512, ddim_steps=50, batch=4, control=False, pa=False, anime=False, f_img=83.63,
            name="configs[1]: 512x512, SeeCoder-v1-0 + SD-v1.5 UNet shapes, 50 DDIM steps, batch 4"),
    3: dict(res=512, ref_res=512, ddim_steps=50, batch=8, control=False, pa=False, anime=True, f_img=83.53,
            name="configs[2]: 512x512, 50 DDIM steps, batch 8, zero-padded [77,768] unconditional context"),
    4: dict(res=512, ref_res=512, ddim_steps=50, batch=4, control=True, pa=False, anime=False, f_img=111.34,
            name="configs[3] per-GPU share: 512x512 + ControlNet (binary 512x512 hint), 50 steps, batch 4 per GPU"),
    5: dict(res=768, ref_res=768, ddim_steps=30, batch=4, control=False, pa=True, anime=False, f_img=139.61,
            name="configs[4] per-GPU share: 768x768, SeeCoder-PA, steps=30 (31 evaluations), batch 4 per GPU"),
}


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference_gpu"])
    ap.add_argument("--config", type=int, default=2, choices=sorted(CONFIGS))
    ap.add_argument("--batch", type=int, default=None, help="override the config's per-GPU batch")
    ap.add_argument("--ddim-steps", type=int, default=None)
    ap.add_argument("--split", action="store_true", help="shard ONE request of `batch` images over the ranks")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-reference", action="store_true")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the images of the last timed step to DIR/<name>.npy (float32) for output comparisons")
    a = ap.parse_args()
    cfg = dict(CONFIGS[a.config])
    if a.batch:
        cfg["batch"] = a.batch
    if a.ddim_steps:
        cfg["ddim_steps"] = a.ddim_steps
    a.cfg = cfg
    return a


# ------------------------------------------------------------------------------------------------
class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.gpu = gpu_index
        self.proc = None
        self.path = None

    def start(self):
        try:
            f = tempfile.NamedTemporaryFile("w", suffix=".csv", delete=False)
            self.path = f.name
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"], stdout=f,
                                         stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None
        return self

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        try:
            for line in open(self.path):
                p = [s.strip() for s in line.split(",")]
                if len(p) < 8:
                    continue
                try:
                    sm.append(float(p[1])); mx.append(float(p[2]))
                except ValueError:
                    continue
                for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), p[4:8]):
                    if val.lower().startswith("active"):
                        reasons.add(name)
            os.unlink(self.path)
        except Exception:
            pass
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def host_threads():
    """All host threads for the CPU legs: torchrun exports OMP_NUM_THREADS=1, which made the r1 reference arm run on
    one core at N > 1 (VERDICT r1)."""
    import torch
    n = os.cpu_count() or 1
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        pass
    try:                                   # one thread per physical core: 128 SMT threads ran the fp32 UNet 10x slower
        import psutil                      # than 64 on the r2 GPU box (81.6 s vs 7.9 s per CFG-pair evaluation)
        n = max(1, min(n, psutil.cpu_count(logical=False) or n))
    except Exception:
        pass
    torch.set_num_threads(n)
    return torch.get_num_threads()


def synth_inputs(cfg, rank=0):
    """Seeded synthetic request of a config (SURVEY.md §8d table): reference image, control hint, uncond context."""
    import torch
    g = torch.Generator().manual_seed(100 + rank)
    out = {"img": torch.rand((1, 3, cfg["ref_res"], cfg["ref_res"]), generator=g)}
    if cfg["control"]:
        out["hint"] = (torch.rand((1, 1, cfg["res"], cfg["res"]), generator=g) > 0.9).float().repeat(1, 3, 1, 1)
    if cfg["anime"]:
        ug = 0.5 * torch.randn((1, 77, 768), generator=g)
        out["uncond"] = torch.cat([ug, torch.zeros((1, 148 - 77, 768))], 1)              # app.py:238-241
    return out


def synth_net(cfg):
    """pfd_b200 pipeline with name-seeded synthetic weights (fp32, CPU)."""
    from pfd_b200 import get_model, model_cfg_bank
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet" if cfg["control"] else "pfd_seecoder"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    if cfg["pa"]:
        from pfd_b200.seecoder import PPE_MLP
        pe = PPE_MLP(freq_num=20, freq_max=None, out_channel=768, mlp_layer=3)            # app.py:166-175
        fill_module_(pe, seed=0, prefix="ctx.image.qtransformer.pe_layer.")
        net.ctx["image"].qtransformer.pe_layer = pe
    net.eval()
    return net


class quiet:
    """The reference prints a banner per request and tqdm-logs every DDIM step: silence it inside timed regions."""

    def __enter__(self):
        self.o, self.e = sys.stdout, sys.stderr
        self.f = open(os.devnull, "w")
        sys.stdout, sys.stderr = self.f, self.f
        return self

    def __exit__(self, *a):
        sys.stdout, sys.stderr = self.o, self.e
        self.f.close()


# ------------------------------------------------------------------------------------------------ reference arms
def build_reference(cfg):
    """The UNMODIFIED reference pipeline (tools/ref_harness.py -> oracle/_ref) on the CPU with the
    same synthetic weights (random init skipped: every tensor is overwritten).  Returns (net, RefSampler class) or None."""
    import torch
    import ref_harness as rh
    if not rh.available():
        return None
    cwd = os.getcwd()
    try:
        with quiet():
            net, _ = rh.build_reference_net("pfd_seecoder_with_controlnet" if cfg["control"] else "pfd_seecoder",
                                            fast=True)
        rh.fill_reference_net(net)
        if cfg["pa"]:
            from lib.model_zoo.seecoder import PPE_MLP
            from pfd_b200.weights import fill_module_
            pe = PPE_MLP(freq_num=20, freq_max=None, out_channel=768, mlp_layer=3)
            fill_module_(pe, seed=0, prefix="ctx.image.qtransformer.pe_layer.")
            pe.eval()
            net.ctx["image"].qtransformer.pe_layer = pe
        from lib.model_zoo.ddim import DDIMSampler as RefSampler
    finally:
        os.chdir(cwd)
    return net, RefSampler


def reference_gpu_leg(cfg, steps=2, warmup=1, gpu_index=0):
    """The reference's own modules in PyTorch eager fp16 on this GPU: ctx_encode -> DDIMSampler.sample -> vae_decode of
    the same synthetic request, host image in / host images out, CUDA events; its own clock sample."""
    import torch
    built = build_reference(cfg)
    if built is None:
        return {"unavailable": "reference tree not staged (oracle/_ref missing)"}
    net, RefSampler = built
    net = net.half()
    net.to("cuda")
    B, L = cfg["batch"], cfg["res"] // 8
    inp = synth_inputs(cfg)
    img_host = inp["img"].half().pin_memory()
    out_host = torch.empty((B, 3, cfg["res"], cfg["res"]), dtype=torch.float16).pin_memory()
    hint = inp["hint"].half().cuda() if cfg["control"] else None
    sampler = RefSampler(net)

    def request():
        with torch.no_grad():
            img = img_host.to("cuda", non_blocking=True)
            c = net.ctx_encode(img, which="image").repeat(B, 1, 1)                         # app.py:235
            u = inp["uncond"].half().cuda().repeat(B, 1, 1) if cfg["anime"] else torch.zeros_like(c)
            torch.manual_seed(20)
            x, _ = sampler.sample(steps=cfg["ddim_steps"], x_info={"type": "image"},
                                  c_info={"type": "image", "conditioning": c, "unconditional_conditioning": u,
                                          "unconditional_guidance_scale": 2.0, "control": hint},
                                  shape=[B, 4, L, L], verbose=False, eta=0.0)
            im = net.vae_decode(x, which="image")
            out_host.copy_(im, non_blocking=True)
            return im

    with quiet():
        for _ in range(warmup):
            request()
        torch.cuda.synchronize()
        clocks = ClockSampler(gpu_index).start()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            im = request()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    clk = clocks.stop()
    res = {"value": B * steps / (ms / 1000.0), "unit": "images/s", "ms_per_request": ms / steps, "requests": steps,
           "warmup": warmup,
           "impl": "unmodified reference modules (oracle/_ref), torch %s eager fp16, no xformers" % torch.__version__,
           "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30, "clocks": clk,
           "output_finite": bool(torch.isfinite(im.float()).all().item())}
    del net, sampler
    torch.cuda.empty_cache()
    return res


def cpu_reference_leg(cfg, max_unet_evals=1):
    """The reference's CPU path (fp32, all host threads) on a bounded sample of the workload: `max_unet_evals`
    CFG-pair UNet(+ControlNet) evaluations of ONE image at the config's latent size, one VAE decode, one SeeCoder
    encode; images/s = 1 / (evals * unet + vae + see / B).  Unmodified reference modules when the staged copy exists
    (kind "reference"), else the oracle port (kind "port")."""
    import torch
    cores = host_threads()
    L, R, B = cfg["res"] // 8, cfg["ref_res"], cfg["batch"]
    evals = len(range(0, 1000, 1000 // cfg["ddim_steps"]))                              # steps=30 -> 31
    g = torch.Generator().manual_seed(0)
    x = torch.randn((1, 4, L, L), generator=g)
    c = 0.5 * torch.randn((1, 148, 768), generator=g)
    z = torch.randn((1, 4, L, L), generator=g)
    inp = synth_inputs(cfg)
    x_in, c_in = torch.cat([x, x]), torch.cat([torch.zeros_like(c), c])
    t = torch.tensor([981, 981])
    built = build_reference(cfg)
    with torch.no_grad():
        if built is not None:
            kind = "reference"
            net, _ = built
            net.device = "cpu"
            c_info = {"type": "image", "c": c_in, "control": inp.get("hint")}
            with quiet():
                t0 = time.perf_counter()
                for _ in range(max_unet_evals):
                    net.apply_model({"type": "image", "x": x_in}, t, c_info)
                t_unet = (time.perf_counter() - t0) / max_unet_evals
                t0 = time.perf_counter(); net.vae_decode(z, which="image"); t_vae = time.perf_counter() - t0
                t0 = time.perf_counter(); net.ctx_encode(inp["img"], which="image"); t_see = time.perf_counter() - t0
        else:
            kind = "port"
            from oracle import pfd_oracle as O
            net = synth_net(cfg)
            sd = {k: v.detach().float() for k, v in net.state_dict().items()}
            usd, vsd, ssd = O.sub(sd, "diffuser.image."), O.sub(sd, "vae.image."), O.sub(sd, "ctx.image.")
            t0 = time.perf_counter()
            for _ in range(max_unet_evals):
                ctl = None
                if cfg["control"]:
                    ctl = O.controlnet_apply(O.sub(sd, "ctl."), O.CONTROLNET_SD15, x_in, inp["hint"], t, c_in)
                O.unet_apply(usd, O.UNET_SD15, x_in, t, c_in, ctl)
            t_unet = (time.perf_counter() - t0) / max_unet_evals
            t0 = time.perf_counter(); O.vae_decode(vsd, O.VAE_SD, z); t_vae = time.perf_counter() - t0
            t0 = time.perf_counter(); O.seecoder_encode(ssd, inp["img"]); t_see = time.perf_counter() - t0
    spi = evals * t_unet + t_vae + t_see / B
    sample = (f"{max_unet_evals} CFG-pair UNet{'+ControlNet' if cfg['control'] else ''} eval(s) of 1 image at {L}x{L} latents "
              f"= {t_unet:.2f}s each; 1 VAE decode {t_vae:.2f}s; 1 SeeCoder encode ({R}x{R}) {t_see:.2f}s; fp32; "
              f"images/s = 1/({evals}*unet + vae + see/{B})")
    return {"value": 1.0 / spi, "unit": "images/s", "cores": cores, "kind": kind, "sample": sample}


def run_reference(args):
    """--impl reference: the reference's own CPU implementation on the host cores, bounded sample (contract ④)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cfg = args.cfg
    cb = cpu_reference_leg(cfg, max_unet_evals=max(1, min(args.steps, 3)))
    value = cb["value"]
    line = {"impl": "reference", "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": cfg["batch"] * 1000.0 / value,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "config": {"workload": cfg["name"] + ", CFG 2.0 - reference CPU path on the host cores (bounded sample, extrapolated)",
                       "config_id": args.config},
            "cpu_baseline": cb,
            "e2e": {"value": value, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


def run_reference_gpu(args):
    """--impl reference_gpu: only the same-GPU PyTorch eager fp16 run of the unmodified reference (context arm)."""
    import torch
    if int(os.environ.get("RANK", "0")) != 0:
        return
    torch.cuda.set_device(0)
    r = reference_gpu_leg(args.cfg, steps=max(1, args.steps), warmup=max(1, min(args.warmup, 1)))
    print(json.dumps({"impl": "reference_gpu", "metric": METRIC,
                      "config": {"workload": args.cfg["name"], "config_id": args.config}, **r}), flush=True)


# ------------------------------------------------------------------------------------------------
def gemm_roofline_pass(net, cfg, cond, uncond, hint):
    """Device time of the dominant kernel (pfd_gemm_f16 = wgmma GEMM / implicit-GEMM conv) inside ONE
    CFG-pair UNet(+ControlNet) evaluation, measured live with CUDA events and without host-launch gaps: the
    evaluation is captured into a CUDA graph twice - once complete, once with every pfd_gemm_f16 launch elided - and
    both graphs are replayed back to back; kernel time = T_full - T_without.
    Algorithmic FLOPs = sum over launches of 2 * rows * N * K from the call descriptors.
    Returns (total_flops, gemm_ms, launches, breakdown_ms)."""
    import torch
    from pfd_b200 import native as nv
    B, L = cfg["batch"], cfg["res"] // 8
    c_full = torch.cat([uncond, cond])
    prep = net.prepare_context(c_full, "image")
    if hint is not None:
        prep["hint"] = net.ctl.hint_features(hint)
    x = torch.randn((B, 4, L, L), device="cuda", dtype=torch.float16)
    t_in = torch.full((2 * B,), 501, device="cuda", dtype=torch.long)
    c_info = {"type": "image", "c": prep["c"], "_pfd_prepared": prep, "control": hint}

    def run():
        return net.apply_model({"type": "image", "x": torch.cat([x, x])}, t_in, c_info)

    stats = {"flops": 0.0, "n": 0}
    orig = {"gemm_raw": nv.gemm_raw}

    def counting(segs, **kw):
        stats["flops"] += 2.0 * kw["W"] * kw["H"] * kw["NB"] * kw["N"] * sum(t * c for (_, t, c, _) in segs)
        stats["n"] += 1
        orig["gemm_raw"](segs, **kw)

    run()
    torch.cuda.synchronize()
    nv.gemm_raw = counting
    try:
        run()
    finally:
        nv.gemm_raw = orig["gemm_raw"]
    torch.cuda.synchronize()

    def graph_ms(skip=()):
        skip = tuple(skip) + (("flash_attn_strided",) if "flash_attn" in skip else ())
        saved = {k: getattr(nv, k) for k in skip}
        try:
            if "gemm_raw" in skip:
                nv.gemm_raw = lambda segs, **kw: None
            if "flash_attn" in skip:
                nv.flash_attn = lambda q, k, vt, **kw: kw["out"]
                nv.flash_attn_strided = lambda q, k, vt, **kw: kw["out"]
            if "groupnorm" in skip:
                def gn(x_, g_, b_, eps_, silu=False, x2=None, groups=32, out=None, **_k):
                    if out is not None:
                        return out
                    c2 = x2.shape[3] if x2 is not None else 0
                    return torch.empty(x_.shape[:3] + (x_.shape[3] + c2,), device=x_.device, dtype=torch.float16)
                nv.groupnorm = gn
            if "layernorm" in skip:
                nv.layernorm = lambda x_, g_, b_, eps_=1e-5, residual=None, out=None: (out if out is not None else torch.empty_like(x_))
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                run()
        finally:
            for k, v in saved.items():
                setattr(nv, k, v)
        for _ in range(10):                  # bring the clocks to the sustained (power-capped) state first
            g.replay()
        torch.cuda.synchronize()
        reps = 25
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    t_full = graph_ms()
    t_nogemm = graph_ms(("gemm_raw",))
    br = {"unet_eval_ms": t_full, "gemm_ms": t_full - t_nogemm}
    try:
        br["flash_attn_ms"] = t_full - graph_ms(("flash_attn",))
        br["groupnorm_ms"] = t_full - graph_ms(("groupnorm",))
        br["layernorm_ms"] = t_full - graph_ms(("layernorm",))
    except Exception as e:  # breakdown is informational only
        br["breakdown_error"] = str(e)
    return stats["flops"], max(t_full - t_nogemm, 1e-6), stats["n"], br


def run_ours(args):
    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from pfd_b200 import DDIMSampler, native as nv, parallel as par
    nv.load()
    cfg = args.cfg
    net = synth_net(cfg).half()
    net.to("cuda")
    if cfg["pa"]:
        net.ctx["image"].qtransformer.pe_layer.cuda()
    B, L, R = cfg["batch"], cfg["res"] // 8, cfg["res"]
    split = args.split and world > 1
    inp = synth_inputs(cfg, rank=0 if split else rank)
    img_host = inp["img"].half().pin_memory()
    img_dev = img_host.cuda()
    hint = inp["hint"].half().cuda() if cfg["control"] else None
    ug = inp["uncond"].half().cuda() if cfg["anime"] else None
    b0, b1 = par.shard_range(B, world, rank) if split else (0, B)
    Bl = b1 - b0                                                          # images this rank samples
    out_host = torch.empty((B, 3, R, R), dtype=torch.float16).pin_memory()
    sampler = DDIMSampler(net, use_cuda_graph=not args.no_graph)

    def request(img):
        if split:
            # rank 0 encodes, conditioning is broadcast; full-batch randn with the request seed, this rank's slice
            c1 = net.ctx_encode(img, "image") if rank == 0 else None
            c1 = par.broadcast_conditioning(c1, 0, shape=(1, 148, 768), dtype=torch.float16, device="cuda")
            xt = par.sharded_noise([B, 4, L, L], seed=20, rank=rank, world=world, device="cuda", dtype=torch.float16)
            x_info = {"type": "image", "xt": xt}
        else:
            c1 = net.ctx_encode(img, "image")                            # app.py:235
            torch.manual_seed(20 + rank)                                 # app.py:259-260
            x_info = {"type": "image"}
        c = c1.repeat(Bl, 1, 1)
        u = ug.repeat(Bl, 1, 1) if ug is not None else torch.zeros_like(c)   # app.py:236-241
        x, _ = sampler.sample(steps=cfg["ddim_steps"], x_info=x_info,
                              c_info={"type": "image", "conditioning": c, "unconditional_conditioning": u,
                                      "unconditional_guidance_scale": 2.0, "control": hint},
                              shape=[Bl, 4, L, L], verbose=False, eta=0.0)
        im = net.vae_decode(x, "image")
        if split:
            im = par.gather_images(im, B)
        return im, c, u

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    for _ in range(max(args.warmup, 1)):
        im, cond, uncond = request(img_dev)
    sync_all()
    clocks = ClockSampler(local).start()
    n0 = nv.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        im, cond, uncond = request(img_dev)
    e1.record()
    sync_all()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"images": im})
    launches = nv.launch_count() - n0
    ms = e0.elapsed_time(e1)
    clk = clocks.stop()
    # ---- e2e: host buffers, H2D of the reference image and D2H of the decoded images every step
    sync_all()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e2.record()
    for _ in range(args.steps):
        dev = img_host.to("cuda", non_blocking=True)
        im, _, _ = request(dev)
        out_host.copy_(im, non_blocking=True)
    e3.record()
    sync_all()
    ms_e2e = e2.elapsed_time(e3)
    if world > 1:
        tt = torch.tensor([ms, ms_e2e], device="cuda", dtype=torch.float64)
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        ms, ms_e2e = tt.tolist()
    n_img = B if split else world * B                                    # images produced per step by the whole job
    value = n_img * args.steps / (ms / 1000.0)
    e2e = n_img * args.steps / (ms_e2e / 1000.0)
    finite = bool(torch.isfinite(im.float()).all().item())

    # ---- informational: device time of the three stages of one request (outside the timed regions)
    stage_ms = None
    if rank == 0 and not split:
        def timed(fn, reps=3):
            fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                r = fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / reps, r
        t_ctx, c1 = timed(lambda: net.ctx_encode(img_dev, "image"))
        cB = c1.repeat(B, 1, 1)
        uB = ug.repeat(B, 1, 1) if ug is not None else torch.zeros_like(cB)
        t_smp, (xs, _) = timed(lambda: sampler.sample(
            steps=cfg["ddim_steps"], x_info={"type": "image"},
            c_info={"type": "image", "conditioning": cB, "unconditional_conditioning": uB,
                    "unconditional_guidance_scale": 2.0, "control": hint},
            shape=[B, 4, L, L], verbose=False, eta=0.0), reps=2)
        t_vae, _ = timed(lambda: net.vae_decode(xs, "image"))
        stage_ms = {"seecoder_encode": t_ctx, "ddim_sampling": t_smp, "vae_decode": t_vae}

    if rank == 0:
        peak_t = 989.0
        which = "H100 SXM data sheet, dense fp16 tensor (700 W card; not a measured rate)"
        roofline = None
        if not split:
            flops, gms, nl, breakdown = gemm_roofline_pass(net, cfg, cond[:B], uncond[:B], hint)
            achieved = flops / (gms / 1000.0) / 1e12 if gms > 0 else 0.0
            evals = len(range(0, 1000, 1000 // cfg["ddim_steps"]))
            if stage_ms is not None:
                breakdown["sampler_overhead_ms"] = stage_ms["ddim_sampling"] - evals * breakdown["unet_eval_ms"]
            roofline = {"bound": "tensor", "kernel": "pfd::gemm_wgmma_kernel<BN> (wgmma GEMM / implicit-GEMM conv)",
                        "achieved": achieved, "peak": peak_t, "unit": "TFLOP/s", "frac": achieved / peak_t,
                        "peak_source": which, "launches_in_unet_eval": nl,
                        "algorithmic_gflop_in_unet_eval": flops / 1e9, "kernel_ms_in_unet_eval": gms,
                        "how": "CUDA events around graph replays of one CFG-pair UNet eval, with minus without the kernel's launches",
                        "unet_eval_breakdown_ms": breakdown,
                        "pipeline_frac": (value / world) * cfg["f_img"] / peak_t}
        gpu_ref = None
        vs_baseline = None
        if world == 1 and not args.no_gpu_reference:
            try:
                gpu_ref = reference_gpu_leg(cfg, steps=2, warmup=1, gpu_index=local)
                if "value" in gpu_ref:
                    vs_baseline = e2e / gpu_ref["value"]
            except Exception as e:  # never lose our own line because the reference arm failed
                gpu_ref = {"unavailable": f"{type(e).__name__}: {e}"[:300]}
        cpu_baseline = None
        if world == 1 and not args.no_cpu_baseline:
            try:
                cpu_baseline = cpu_reference_leg(cfg)
            except Exception as e:
                cpu_baseline = {"unavailable": f"{type(e).__name__}: {e}"[:300]}
        line = {"metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
                "scaling": "strong" if split else "weak",
                "vs_baseline": vs_baseline,
                "vs_baseline_source": None if vs_baseline is None else
                "e2e / gpu_reference.value: the UNMODIFIED reference (torch eager fp16) timed on this GPU in this run; "
                "BASELINE.md publishes no number (the north-star's x2 target is against this arm)",
                "dtype": "fp16", "data": "synthetic",
                "config": {"workload": cfg["name"] + ", CFG 2.0, fp16", "config_id": args.config,
                           "global_batch": n_img, "batch_per_gpu": Bl,
                           "parallelism": (f"dp{world}: ONE request of {B} images sharded (parallel.py: rank-0 encode + broadcast, "
                                           "full-batch randn + slice, all-gather of images)") if split else
                                          f"dp{world} (one request of {B} images per GPU, no data-path collective)",
                           "l2": "working set (1.7 GB weights + GBs of activations per step) is larger than the 50 MB L2",
                           "cuda_graph": False if args.no_graph else f"all {cfg['ddim_steps']} DDIM steps in one captured graph"},
                "roofline": roofline, "cpu_baseline": cpu_baseline, "gpu_reference": gpu_ref,
                "e2e": {"value": e2e, "unit": "images/s", "h2d_bytes_per_step": img_host.numel() * 2,
                        "d2h_bytes_per_step": out_host.numel() * 2},
                "gpu_launches": int(launches), "clocks": clk, "output_finite": finite, "stage_ms": stage_ms}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(dirname, arrays):
    """Each array -> DIR/<name>.npy as float32.  An array above the size limit is replaced by a fixed, seeded sample of
    its flattened elements (<name>_sample.npy) with their flat indices (<name>_sample_index.npy, float64)."""
    import numpy as np
    os.makedirs(dirname, exist_ok=True)
    per = DUMP_LIMIT_BYTES // max(1, len(arrays))
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy()
        if a.nbytes <= per:
            np.save(os.path.join(dirname, f"{name}.npy"), a)
            continue
        n = per // 12                                                     # 4 B value + 8 B index per element
        idx = np.sort(np.random.default_rng(0).choice(a.size, size=n, replace=False))
        np.save(os.path.join(dirname, f"{name}_sample.npy"), a.reshape(-1)[idx])
        np.save(os.path.join(dirname, f"{name}_sample_index.npy"), idx.astype(np.float64))


def main():
    args = parse()
    if args.gpus > 1 and "WORLD_SIZE" not in os.environ:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={args.gpus}",
               "--master-addr", "127.0.0.1", "--master-port", "29517", os.path.abspath(__file__)] + sys.argv[1:]
        sys.exit(subprocess.call(cmd))
    if args.impl == "reference":
        run_reference(args)
    elif args.impl == "reference_gpu":
        run_reference_gpu(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
