"""Cross-process reproducibility in deterministic mode: one small request (SeeCoder context of a seeded image, DDIM with
CFG and ControlNet at 16x16 latents, VAE decode) on the synthetic-weight pfd_seecoder_with_controlnet net, printed as
SHA-256 hashes of the context, the final latent and the decoded images.  Two runs of the same build on the same GPU
architecture must print the same line.

    python tools/determinism_check.py [--default]      # --default: run in the default mode instead
    python tools/determinism_check.py --samplers       # also hash every sampling-loop mode of both samplers

--samplers adds one SAMPLER_RESULT line per case of SAMPLER_CASES: the SHA-256 of the final latent and of the stacked
intermediates (log_every_t=1), and the library launch count, of two sample() calls on one sampler object (the first
builds and captures the loop, the second replays it).  Unseeded cases reset torch's generator before each call, so two
builds that run the same kernels with the same noise print the same lines.
"""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sha256(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


# name -> sampler ("ddim" or a Sampler type), options: eta, seeded, graph (False = eager), spg (DDIM steps_per_graph),
# img2img, temperature, guidance, control, big (64x64 latents, batch 4, 50 DDIM steps: the size of bench.py's config 2)
SAMPLER_CASES = {
    "ddim_eta0": ("ddim", {}),
    "ddim_eta0_spg4": ("ddim", {"spg": 4}),
    "ddim_eta0_spg1": ("ddim", {"spg": 1}),
    "ddim_eta0_eager": ("ddim", {"graph": False}),
    "ddim_eta0.5": ("ddim", {"eta": 0.5}),
    "ddim_eta0.5_eager": ("ddim", {"eta": 0.5, "graph": False}),
    "ddim_eta0.5_seeded": ("ddim", {"eta": 0.5, "seeded": True}),
    "ddim_eta0.5_seeded_eager": ("ddim", {"eta": 0.5, "seeded": True, "graph": False}),
    "ddim_img2img": ("ddim", {"eta": 0.5, "img2img": True}),
    "ddim_img2img_seeded": ("ddim", {"eta": 0.5, "img2img": True, "seeded": True}),
    "ddim_eta0.5_temp0.5": ("ddim", {"eta": 0.5, "temperature": 0.5}),
    "ddim_eta0.5_temp0.5_seeded": ("ddim", {"eta": 0.5, "temperature": 0.5, "seeded": True}),
    "ddim_no_cfg": ("ddim", {"guidance": 1.0}),
    "dpmpp_2m_no_cfg": ("dpmpp_2m", {"guidance": 1.0}),
    "euler_a_eta0": ("euler_a", {"eta": 0.0}),
    "euler_a_eta0_seeded": ("euler_a", {"eta": 0.0, "seeded": True}),
    "euler_a_eta1": ("euler_a", {"eta": 1.0}),
    "euler_a_eta1_seeded": ("euler_a", {"eta": 1.0, "seeded": True}),
    "dpmpp_2m": ("dpmpp_2m", {}),
    "dpmpp_2m_sde": ("dpmpp_2m_sde", {"eta": 1.0}),
    "dpmpp_2m_sde_seeded": ("dpmpp_2m_sde", {"eta": 1.0, "seeded": True}),
    "ddim_control": ("ddim", {"control": True}),
    "euler_a_eta1_control": ("euler_a", {"eta": 1.0, "control": True}),
    "ddim50_64x64_b4_eta0": ("ddim", {"big": True}),
    "ddim50_64x64_b4_eta1": ("ddim", {"eta": 1.0, "big": True}),
}


def sampler_rows(net, inp):
    from oracle.golden_inputs import seeded
    from pfd_b200 import DDIMSampler, Sampler
    from pfd_b200 import native as nv
    for name, (kind, o) in SAMPLER_CASES.items():
        B, lat, steps = (4, 64, 50) if o.get("big") else (2, 16, 8)
        cond = seeded((B, 148, 768), 16, 0.5).cuda().half()
        c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
                  "unconditional_guidance_scale": o.get("guidance", 2.0),
                  "control": inp["hint"].cuda().half() if o.get("control") else None}
        x_info = {"type": "image"}
        if o.get("seeded"):
            x_info["seeds"] = 1000
        if o.get("img2img"):
            x_info.update(x0=seeded((B, 4, lat, lat), 17).cuda().half(), x0_forward_timesteps=5)
        graph = o.get("graph", True)
        if kind == "ddim":
            smp = DDIMSampler(net, use_cuda_graph=graph, steps_per_graph=o.get("spg"))
            kw = {"eta": o.get("eta", 0.0), "temperature": o.get("temperature", 1.0), "verbose": False}
        else:
            smp = Sampler(net, type=kind, use_cuda_graph=graph)
            kw = {"eta": o.get("eta", 1.0)}
        row = {"case": name}
        for call in (1, 2):
            torch.manual_seed(0)
            n0 = nv.launch_count()
            x, inter = smp.sample(steps=steps, shape=[B, 4, lat, lat], x_info=dict(x_info), c_info=dict(c_info),
                                  log_every_t=1, **kw)
            torch.cuda.synchronize()
            row[f"launches{call}"] = nv.launch_count() - n0
            row[f"latent{call}"] = sha256(x)
            row[f"pred_xt{call}"] = sha256(torch.stack(inter["pred_xt"]))
            row[f"pred_x0{call}"] = sha256(torch.stack(inter["pred_x0"]))
        print("SAMPLER_RESULT " + json.dumps(row), flush=True)
        del smp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--default", action="store_true", help="run in the default (non-deterministic) mode")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--samplers", action="store_true", help="also hash every sampling-loop mode (SAMPLER_CASES)")
    args = ap.parse_args()
    from oracle.golden_inputs import golden_inputs
    from pfd_b200 import DDIMSampler, get_model, is_deterministic, model_cfg_bank, set_deterministic
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    set_deterministic(not args.default)
    net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    net.eval()
    inp = golden_inputs()
    B = 2
    ctx = net.ctx_encode(inp["img"].cuda(), "image")
    cond = ctx.repeat(B, 1, 1)
    xt = torch.cat([inp["x_T"], -inp["x_T"]]).cuda().half()
    x, _ = DDIMSampler(net).sample(steps=args.steps, shape=[B, 4, 16, 16], x_info={"type": "image", "xt": xt},
                                   c_info={"type": "image", "conditioning": cond,
                                           "unconditional_conditioning": torch.zeros_like(cond),
                                           "unconditional_guidance_scale": 2.0, "control": inp["hint"].cuda().half()},
                                   verbose=False, eta=0.0)
    im = net.vae_decode(x, "image")
    torch.cuda.synchronize()
    res = {"deterministic": is_deterministic(), "device": torch.cuda.get_device_name(),
           "context": sha256(ctx), "latent": sha256(x), "images": sha256(im)}
    print("DETERMINISM_RESULT " + json.dumps(res), flush=True)
    if args.samplers:
        sampler_rows(net, inp)


if __name__ == "__main__":
    main()
