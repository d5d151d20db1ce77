"""Cross-process reproducibility in deterministic mode: one small request (SeeCoder context of a seeded image, DDIM with
CFG and ControlNet at 16x16 latents, VAE decode) on the synthetic-weight pfd_seecoder_with_controlnet net, printed as
SHA-256 hashes of the context, the final latent and the decoded images.  Two runs of the same build on the same GPU
architecture must print the same line.

    python tools/determinism_check.py [--default]      # --default: run in the default mode instead
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--default", action="store_true", help="run in the default (non-deterministic) mode")
    ap.add_argument("--steps", type=int, default=4)
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


if __name__ == "__main__":
    main()
