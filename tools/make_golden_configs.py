"""Golden outputs of the UNMODIFIED reference at the BASELINE configs' own sizes (VERDICT r1 item 1).

Runs only where the reference tree exists (build container: /root/reference).  The reference pipeline is built
through its own registry (tools/ref_harness.py), filled with the name-seeded synthetic weights, and run in fp32 on
the CPU on the seeded inputs of oracle/golden_inputs.config_inputs(); the outputs are stored (fp16 where large)
in tests/golden/config_outputs.npz and compared against the CUDA path by tests/test_configs_gpu.py.

    python tools/make_golden_configs.py [case ...]      # ~10 min on 8 cores; cases: c1 .. c9
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLD = os.path.join(ROOT, "tests", "golden")
OUT = os.path.join(GOLD, "config_outputs.npz")

import ref_harness as rh  # noqa: E402
from oracle.golden_inputs import config_inputs  # noqa: E402
from pfd_b200.weights import fill_module_  # noqa: E402


class patched:
    """Temporarily replace torch.randn / torch.randn_like by a queue of prepared tensors."""

    def __init__(self, randn=None, randn_like=None):
        self.q, self.ql = list(randn or []), list(randn_like or [])

    def __enter__(self):
        self.r, self.rl = torch.randn, torch.randn_like
        if self.q:
            torch.randn = lambda *a, **k: self.q.pop(0).clone()
        if self.ql:
            torch.randn_like = lambda x, *a, **k: self.ql.pop(0).clone().to(x.dtype)
        return self

    def __exit__(self, *e):
        torch.randn, torch.randn_like = self.r, self.rl


def sub(t, stride):
    return t.detach().float().reshape(-1)[::stride].numpy().astype(np.float32)


# Tensors the tests feed back into the pipeline (teacher forcing, decode of the reference latent, the posterior
# formula) are stored whole; every other tensor is only compared, so a fixed strided sample of at most
# SAMPLE_MAX elements is stored with its full shape under "<key>__shape" (keeps the file under 1 MB).
FULL_KEYS = ("c1_latent", "c5_ctx", "c5_x_step0", "c7_latent", "c8_mean", "c8_logvar", "c9_latent")
SAMPLE_MAX = 4096


def sample_for_storage(out):
    res = {}
    for k, v in out.items():
        if k.endswith("__shape") or k in FULL_KEYS:
            res[k] = v
            continue
        v = np.asarray(v)
        stride = -(-v.size // SAMPLE_MAX)
        res[k] = v.reshape(-1)[::stride].astype(np.float32)
        res[k + "__shape"] = np.asarray(v.shape, dtype=np.int64)
    return res


def main():
    cases = sys.argv[1:] or ["c1", "c2", "c3", "c4", "c5", "c6", "c7", "c8", "c9"]
    torch.set_grad_enabled(False)
    out = dict(np.load(OUT)) if os.path.exists(OUT) else {}
    t0 = time.time()
    net, _ = rh.build_reference_net()
    rh.fill_reference_net(net)
    net.device = "cpu"
    print(f"reference net ready in {time.time() - t0:.0f}s", flush=True)
    inp = config_inputs()
    sampler = rh.cpu_sampler(net)

    def eps(x, t, c, control=None):
        tt = torch.full((x.shape[0],), int(t), dtype=torch.long)
        return net.apply_model({"type": "image", "x": x}, tt, {"type": "image", "c": c, "control": control})

    if "c1" in cases:
        t1 = time.time()
        ctx = net.ctx_encode(inp["c1_img"], "image")
        with patched(randn=[inp["c1_xT"]]):
            x, _ = sampler.sample(steps=10, x_info={"type": "image"},
                                  c_info={"type": "image", "conditioning": ctx,
                                          "unconditional_conditioning": torch.zeros_like(ctx),
                                          "unconditional_guidance_scale": 2.0, "control": None},
                                  shape=[1, 4, 64, 64], verbose=False, eta=0.0)
        im = net.vae_decode(x, "image")
        out.update(c1_ctx=ctx.numpy().astype(np.float16), c1_latent=x.numpy().astype(np.float32),
                   c1_image=im.numpy().astype(np.float16))
        print(f"c1 done {time.time() - t1:.0f}s: latent rms {x.pow(2).mean().sqrt():.3f} image mean {im.mean():.3f}", flush=True)

    if "c2" in cases:
        t1 = time.time()
        x = torch.cat([inp["c2_x"]] * 2)
        cond = inp["c2_cond"].repeat(4, 1, 1)
        c = torch.cat([torch.zeros_like(cond), cond])
        for t in inp["c2_t"]:
            e = eps(x, t, c)
            out[f"c2_eps_t{t}"] = e.numpy().astype(np.float32)
            print(f"c2 t={t}: eps rms {e.pow(2).mean().sqrt():.3f}", flush=True)
        print(f"c2 done {time.time() - t1:.0f}s", flush=True)

    if "c3" in cases:
        x = torch.cat([inp["c3_x"]] * 2)
        cond = inp["c3_cond"].repeat(2, 1, 1)
        c = torch.cat([inp["c3_uncond"].repeat(2, 1, 1), cond])
        e = eps(x, inp["c3_t"], c)
        out["c3_eps"] = e.numpy().astype(np.float32)
        print(f"c3: eps rms {e.pow(2).mean().sqrt():.3f}", flush=True)

    if "c4" in cases:
        x = torch.cat([inp["c4_x"]] * 2)
        cond = inp["c4_cond"].repeat(2, 1, 1)
        c = torch.cat([torch.zeros_like(cond), cond])
        tt = torch.full((4,), int(inp["c4_t"]), dtype=torch.long)
        ctl = net.ctl(x, hint=inp["c4_hint"], timesteps=tt, context=c)
        for i, o in enumerate(ctl):
            out[f"c4_ctl_{i}_sub"] = sub(o, 97)
        e = eps(x, inp["c4_t"], c, control=inp["c4_hint"])
        out["c4_eps"] = e.numpy().astype(np.float32)
        print(f"c4: eps rms {e.pow(2).mean().sqrt():.3f}", flush=True)

    if "c5" in cases or "c6" in cases:
        enc = net.ctx["image"]
        if "c6" in cases:
            fea = enc.imencoder(inp["c6_img"])
            for k in ("res3", "res4", "res5"):
                out[f"c6_swin_{k}_sub"] = sub(fea[k], 31)
            ctx = net.ctx_encode(inp["c6_img"], "image")
            out["c6_ctx"] = ctx.numpy().astype(np.float16)
            print(f"c6: ctx rms {ctx.pow(2).mean().sqrt():.3f}", flush=True)
        if "c5" in cases:
            t1 = time.time()
            from lib.model_zoo.seecoder import PPE_MLP
            pe = PPE_MLP(freq_num=20, freq_max=None, out_channel=768, mlp_layer=3)             # app.py:166-175
            fill_module_(pe, seed=0, prefix="ctx.image.qtransformer.pe_layer.")
            pe.eval()
            enc.qtransformer.pe_layer = pe
            try:
                ctx = net.ctx_encode(inp["c5_img"], "image")
            finally:
                enc.qtransformer.pe_layer = None
            out["c5_ctx"] = ctx.numpy().astype(np.float16)
            sampler.make_schedule(ddim_num_steps=30, ddim_eta=0.0, verbose=False)
            ts = sampler.ddim_timesteps
            assert len(ts) == 31
            total = len(ts)
            x_info = {"type": "image", "x": inp["c5_xT"]}
            c_info = {"type": "image", "conditioning": ctx, "unconditional_conditioning": torch.zeros_like(ctx),
                      "unconditional_guidance_scale": 2.0, "control": None}
            for i in range(2):
                index = total - i - 1
                tt = torch.full((1,), int(ts[index]), dtype=torch.long)
                x_prev, p0 = sampler.p_sample_ddim(x_info, c_info, tt, index)
                out[f"c5_x_step{i}"] = x_prev.numpy().astype(np.float32)
                out[f"c5_x0_step{i}"] = p0.numpy().astype(np.float32)
                x_info["x"] = x_prev
            print(f"c5 done {time.time() - t1:.0f}s: x rms {x_prev.pow(2).mean().sqrt():.3f}", flush=True)

    if "c7" in cases:
        cond = inp["c7_cond"]
        with patched(randn=[inp["c7_xT"]], randn_like=inp["c7_noise"]):
            x, _ = sampler.sample(steps=4, x_info={"type": "image"},
                                  c_info={"type": "image", "conditioning": cond,
                                          "unconditional_conditioning": torch.zeros_like(cond),
                                          "unconditional_guidance_scale": 2.0, "control": None},
                                  shape=[1, 4, 16, 16], verbose=False, eta=0.5)
        out["c7_latent"] = x.numpy().astype(np.float32)
        print(f"c7: latent rms {x.pow(2).mean().sqrt():.3f}", flush=True)

    if "c8" in cases:
        post = net.vae["image"].encode(inp["c8_img"], out_posterior=True)
        out["c8_mean"] = post.mean.numpy().astype(np.float32)
        out["c8_logvar"] = post.logvar.numpy().astype(np.float32)
        print(f"c8: posterior mean rms {post.mean.pow(2).mean().sqrt():.3f} logvar mean {post.logvar.mean():.3f}", flush=True)

    if "c9" in cases:
        mk = lambda c, r: {"type": "image", "conditioning": c, "unconditional_conditioning": torch.zeros_like(c),
                           "unconditional_guidance_scale": 2.0, "ratio": r}
        with patched(randn=[inp["c9_xT"]]):
            x, _ = sampler.sample_multicontext(steps=4, x_info={"type": "image"},
                                               c_info_list=[mk(inp["c9_cond_a"], 0.3), mk(inp["c9_cond_b"], 0.7)],
                                               shape=[1, 4, 16, 16], verbose=False, eta=0.0)
        out["c9_latent"] = x.numpy().astype(np.float32)
        print(f"c9: latent rms {x.pow(2).mean().sqrt():.3f}", flush=True)

    np.savez_compressed(OUT, **sample_for_storage(out))
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB) in {time.time() - t0:.0f}s", flush=True)


if __name__ == "__main__":
    main()
