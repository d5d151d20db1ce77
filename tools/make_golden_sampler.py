"""Write tests/golden/sampler_reference.npz from the UNMODIFIED reference sampler (lib/model_zoo/sampler.py).

The reference module is imported through tools/ref_harness.py.  Its `Sampler` only needs `net.alphas_cumprod` for the
schedule and `net.apply_model(x, sigma)` as a denoiser, so a stub net supplies both:
  - alphas_cumprod: the pfd schedule (pfd.yaml: linear 0.00085 -> 0.012, 1000 steps) in fp32 and rounded to fp16
    (what net.half() leaves in the buffer);
  - apply_model: the exact denoiser for Gaussian data N(mu, s^2), D = (s^2 x + sigma^2 mu) / (s^2 + sigma^2).
Stored: `sigmas_{n}_{fp32|fp16}` = Sampler.get_sigmas(n) for n in {1, 10, 20, 25, 50}; and per Euler-ancestral case i
(`ea_{i}_case` = [seed, n, fp16?], eta = 1, the reference default): the starting unit noise drawn after
torch.manual_seed(seed), the sigmas, every x the loop evaluated the denoiser at (`ea_{i}_xs`) and the result.

    python tools/make_golden_sampler.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pfd_oracle as PO  # noqa: E402
from tools import ref_harness  # noqa: E402

NS = (1, 10, 20, 25, 50)
SHAPE = (2, 4, 8, 8)
MU_SEED, S = 7, 0.5
EA_CASES = [(21, 10, False), (22, 25, True)]


def gaussian_mu():
    return torch.randn(SHAPE, generator=torch.Generator().manual_seed(MU_SEED))


class StubNet:
    def __init__(self, alphas_cumprod, mu):
        self.alphas_cumprod = alphas_cumprod
        self.mu = mu
        self.xs = []

    def apply_model(self, x, sigma):
        self.xs.append(x.clone())
        sg = sigma.reshape(-1, *([1] * (x.dim() - 1))).to(x.dtype)
        return (S * S * x + sg * sg * self.mu) / (S * S + sg * sg)


def main():
    ref_harness.import_reference()
    from lib.model_zoo.sampler import Sampler

    ac32 = PO.schedule_buffers()["alphas_cumprod"]
    acs = {"fp32": ac32, "fp16": ac32.half()}
    mu = gaussian_mu()
    arrays = {"gauss": np.array([MU_SEED, S], np.float64), "shape": np.array(SHAPE, np.int64)}
    for tag, ac in acs.items():
        smp = Sampler(StubNet(ac, mu))
        for n in NS:
            arrays[f"sigmas_{n}_{tag}"] = smp.get_sigmas(n).numpy().astype(np.float64)
    for i, (seed, n, f16) in enumerate(EA_CASES):
        net = StubNet(acs["fp16" if f16 else "fp32"], mu)
        smp = Sampler(net)
        sigmas = smp.get_sigmas(n)
        torch.manual_seed(seed)
        xt = torch.randn(SHAPE)
        x = smp.sample_euler_ancestral(x_info={"x": xt}, c_info=None, sigmas=sigmas)
        arrays[f"ea_{i}_case"] = np.array([seed, n, int(f16)], np.int64)
        arrays[f"ea_{i}_xt"] = xt.numpy()
        arrays[f"ea_{i}_sigmas"] = sigmas.numpy().astype(np.float64)
        arrays[f"ea_{i}_xs"] = torch.stack(net.xs).numpy()
        arrays[f"ea_{i}_out"] = x.numpy()
        print(f"[golden-sampler] euler_a case {i}: n={n} fp16={f16} |x_out| rms {x.pow(2).mean().sqrt():.4f}")
    print("[golden-sampler] last nonzero sigma at n=20: fp32 %.4f, fp16 %.4f"
          % (arrays["sigmas_20_fp32"][-2], arrays["sigmas_20_fp16"][-2]))
    path = os.path.join(ROOT, "tests", "golden", "sampler_reference.npz")
    np.savez_compressed(path, **arrays)
    print(f"[golden-sampler] wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
