"""k-diffusion samplers — Euler ancestral, DPM-Solver++(2M) and DPM-Solver++(2M) SDE — completing
lib/model_zoo/sampler.py.

The reference's `Sampler` (sampler.py:29-104) builds the sigma schedule from `net.alphas_cumprod` (`get_sigmas`,
log-sigma interpolation over t = linspace(999, 0, n), then a zero appended) and holds the Euler-ancestral loop
(`sample_euler_ancestral`, `get_ancestral_step`, `to_d`), but its `sample` never wraps the eps-prediction UNet as a
denoiser and never applies CFG, so it cannot run.  This module supplies the missing wrapper

    c_in = 1 / sqrt(sigma^2 + 1),   eps = CFG(UNet(x * c_in, t(sigma))),   D = x - sigma * eps

with t(sigma) the fractional timestep of the schedule, and runs both samplers with the calling convention of
DDIMSampler:

    x, inter = Sampler(net, type="dpmpp_2m").sample(steps=20, shape=[B, 4, h // 8, w // 8],
                                                     x_info={"type": "image"}, c_info={...})

Every step of either type is x' = a*x + b*D + c*D_prev + u*noise.  The per-step coefficients are computed here in
float64; the update itself is one CUDA kernel (pfd_ksampler_step_f32) that keeps the state in fp32 (sigma_0 * x_T
reaches ~60 and DPM++'s small corrections would be lost in fp16) and writes the next step's fp16 UNet input into both
CFG halves.  The step counter and the float timestep table live on the device (pfd_ksampler_begin_step), so one
captured CUDA graph holds the whole loop when it is deterministic (dpmpp_2m, or euler_a / dpmpp_2m_sde with eta = 0).
A stochastic loop (euler_a or dpmpp_2m_sde with eta > 0) replays a one-step graph per step with the noise drawn on the
host in between, unless the request carries per-sample seeds (x_info["seeds"], pfd_b200/rng.py): then each step's noise
is drawn on the device from the step counter (stream 1, draw = step index) and one graph holds the whole loop too.
The loop engine, shared with DDIMSampler, is loop.py.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import loop
from . import native as nv
from . import rng

TYPES = {"euler_a": "euler_a", "eular_a": "euler_a", "dpmpp_2m": "dpmpp_2m", "dpmpp_2m_sde": "dpmpp_2m_sde"}
STOCHASTIC = ("euler_a", "dpmpp_2m_sde")          # the types whose eta adds noise


def model_log_sigmas(alphas_cumprod: torch.Tensor) -> torch.Tensor:
    """sampler.py:38-39, in the dtype of `alphas_cumprod` (fp16 after net.half(), SURVEY.md App. C #6)."""
    ac = alphas_cumprod.detach().cpu()
    return (((1 - ac) / ac) ** 0.5).log()


def get_sigmas(alphas_cumprod: torch.Tensor, n: int) -> torch.Tensor:
    """sampler.py:41-54 (`t_to_sigma` + `get_sigmas(n)`): n sigmas at t = linspace(T-1, 0, n), then a zero."""
    log_sigmas = model_log_sigmas(alphas_cumprod)
    t = torch.linspace(len(log_sigmas) - 1, 0, n)
    low_idx, high_idx, w = t.floor().long(), t.ceil().long(), t.frac()
    log_sigma = (1 - w) * log_sigmas[low_idx] + w * log_sigmas[high_idx]
    return torch.cat([log_sigma.exp(), torch.zeros(1, dtype=log_sigma.dtype)])


def schedule_timesteps(n: int, num_timesteps: int) -> np.ndarray:
    """The fractional UNet timestep of each sigma of get_sigmas(n): the t it was interpolated at."""
    return torch.linspace(num_timesteps - 1, 0, n).double().numpy()


def sigma_to_t(sigmas, log_sigmas: torch.Tensor) -> np.ndarray:
    """Inverse of the log-sigma interpolation (k-diffusion's DiscreteSchedule.sigma_to_t), in float64."""
    ls = log_sigmas.double().numpy()
    out = []
    for s in np.asarray(sigmas, dtype=np.float64):
        lsig = math.log(s)
        low = min(int(np.sum(lsig - ls >= 0)) - 1, len(ls) - 2)
        low = max(low, 0)
        lo, hi = ls[low], ls[low + 1]
        w = 0.0 if hi == lo else min(max((lo - lsig) / (lo - hi), 0.0), 1.0)
        out.append((1 - w) * low + w * (low + 1))
    return np.asarray(out, dtype=np.float64)


def ancestral_step(sigma_from: float, sigma_to: float, eta: float = 1.0):
    """sampler.py:19-24 (get_ancestral_step): (sigma_down, sigma_up)."""
    if not eta:
        return sigma_to, 0.0
    sigma_up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def coef_table(kind: str, sigmas, eta: float = 1.0) -> np.ndarray:
    """[steps, 6] float64 rows {sigma, a, b, c, u, c_in_next} such that step i is
    x_{i+1} = a*x_i + b*D_i + c*D_{i-1} + u*noise_i, D_i = x_i - sigma_i*eps_i.
      euler_a:  x + (x - D)/sigma * (sigma_down - sigma) + sigma_up*noise (sampler.py:97-103), i.e. a = sigma_down/sigma;
      dpmpp_2m: the DPM-Solver++(2M) multistep rule in log-sigma time, first-order on the first step and on the step
                to sigma = 0;
      dpmpp_2m_sde: k-diffusion's sample_dpmpp_2m_sde (midpoint correction, Gaussian per-step noise): with
                h = ln sigma - ln sigma_next, eta_h = eta*h, phi = -expm1(-h - eta_h):
                a = (sigma_next/sigma) e^-eta_h, b = phi, c = 0, u = sigma_next sqrt(-expm1(-2 eta_h)), and from the
                second step on (r = h_prev/h) b += phi/(2r), c = -phi/(2r); the step to sigma = 0 is x' = D.
                eta = 0 gives dpmpp_2m's table."""
    s = np.asarray(sigmas, dtype=np.float64)
    n = len(s) - 1
    tab = np.zeros((n, nv.PFD_KSAMPLER_NCOEF), dtype=np.float64)
    for i in range(n):
        sig, nxt = s[i], s[i + 1]
        if kind == "euler_a":
            down, up = ancestral_step(sig, nxt, eta)
            a, b, c, u = down / sig, 1.0 - down / sig, 0.0, (up if nxt > 0 else 0.0)
        elif kind == "dpmpp_2m":
            if nxt == 0:
                a, b, c = 0.0, 1.0, 0.0
            else:
                h = math.log(sig) - math.log(nxt)
                phi = -math.expm1(-h)
                a = nxt / sig
                if i == 0:
                    b, c = phi, 0.0
                else:
                    r = (math.log(s[i - 1]) - math.log(sig)) / h
                    b, c = phi * (1 + 1 / (2 * r)), -phi / (2 * r)
            u = 0.0
        elif kind == "dpmpp_2m_sde":
            if nxt == 0:
                a, b, c, u = 0.0, 1.0, 0.0, 0.0
            else:
                h = math.log(sig) - math.log(nxt)
                eta_h = eta * h
                phi = -math.expm1(-h - eta_h)
                a, b, c = nxt / sig * math.exp(-eta_h), phi, 0.0
                u = nxt * math.sqrt(-math.expm1(-2.0 * eta_h))
                if i > 0:
                    r = (math.log(s[i - 1]) - math.log(sig)) / h
                    b, c = b + 0.5 * phi / r, -0.5 * phi / r
        else:
            raise ValueError(f"unknown sampler type {kind!r}")
        tab[i] = (sig, a, b, c, u, 1.0 / math.sqrt(nxt * nxt + 1.0))
    return tab


def log_steps(total: int, log_every_t: int) -> List[int]:
    """Steps whose (UNet input, D) go to `intermediates`: DDIM's rule (ddim.py:122) with schedule index total-1-step."""
    return [k for k in range(total) if (total - 1 - k) % log_every_t == 0 or k == 0]


class Sampler(object):
    """Euler-ancestral ('euler_a', alias 'eular_a') / DPM-Solver++(2M) ('dpmpp_2m') / DPM-Solver++(2M) SDE
    ('dpmpp_2m_sde') sampler for the pfd nets."""

    def __init__(self, net, type="euler_a", **kwargs):
        if type not in TYPES:
            raise ValueError(f"Sampler type {type!r}: expected one of {sorted(TYPES)}")
        self.net = net
        self.type = TYPES[type]
        self.use_cuda_graph = kwargs.get("use_cuda_graph", True)
        self._states = {}

    def get_sigmas(self, n: int) -> torch.Tensor:
        return get_sigmas(self.net.alphas_cumprod, n)

    @torch.no_grad()
    def sample(self, steps, shape, x_info, c_info, eta=1.0, sigmas: Optional[Sequence[float]] = None,
               log_every_t=100, verbose=True):
        """-> (x fp16 NCHW latent for net.vae_decode, {"pred_xt": [...], "pred_x0": [...]}).
        eta: noise scale of euler_a (1 = ancestral, 0 = plain Euler) and dpmpp_2m_sde (0 = dpmpp_2m); ignored by
             dpmpp_2m.
        sigmas: explicit descending schedule (its timesteps by sigma_to_t); default get_sigmas(steps).
        x_info["xt"]: unit noise, scaled by sigma_0 (sampler.py:89); otherwise drawn with torch.randn, or from the
        per-sample seeds x_info["seeds"] (stream 0), which also make the per-step noise come from the device
        (stream 1, draw = step index) inside one graph of the whole loop."""
        model = self.net
        if x_info.get("x0", None) is not None:
            raise NotImplementedError("img2img (x_info['x0']) is only available with DDIMSampler")
        if sigmas is None:
            sig = self.get_sigmas(int(steps)).double().numpy()
            ts = schedule_timesteps(int(steps), int(model.alphas_cumprod.shape[0]))
        else:
            sig = np.asarray([float(s) for s in sigmas], dtype=np.float64)
            if sig.ndim != 1 or len(sig) < 2 or np.any(sig[:-1] <= 0) or np.any(np.diff(sig) >= 0):
                raise ValueError("sigmas must be a descending schedule of at least two values, positive except the last")
            ts = sigma_to_t(sig[:-1], model_log_sigmas(model.alphas_cumprod))
        eta = float(eta) if self.type in STOCHASTIC else 0.0
        total = len(sig) - 1
        coef = coef_table(self.type, sig, eta)
        stochastic = self.type in STOCHASTIC and eta != 0.0

        seeds = loop.request_seeds(x_info, shape[0], model.device)
        xt = loop.initial_noise(x_info, shape, seeds, model.device, model.get_dtype())     # sampler.py:73
        cfg = loop.cfg_context(c_info)
        seeded = seeds is not None
        logs = log_steps(total, log_every_t)
        key = loop.state_key(model, xt, cfg, x_info, c_info, total, logs, stochastic, seeded)
        st = loop.cached_state(self._states, key, self.use_cuda_graph, lambda: _KSamplerState(
            model, tuple(xt.shape), cfg, x_info["type"], c_info["type"], total, logs, stochastic, seeded,
            self.use_cuda_graph))
        st.load_request(xt, float(sig[0]), 1.0 / math.sqrt(sig[0] ** 2 + 1.0), cfg.c_full, cfg.cc,
                        torch.as_tensor(coef, dtype=torch.float32), torch.as_tensor(ts, dtype=torch.float32), seeds)
        # sampler.py:102-103: one randn_like(x) per step with sigma_next > 0 (x is in the net's dtype)
        st.run(sig[1:] > 0)
        return st.result(x_info, c_info, cfg.c_full)


class _KSamplerState(loop.LoopState):
    """fp32 state x, the previous step's denoised D_prev, and the fp16 UNet input / output the update writes; the step
    counter counts up (0, ..., total-1)."""

    T_DTYPE, NCOEF, WARMUP_STEP = torch.float32, nv.PFD_KSAMPLER_NCOEF, -1

    def __init__(self, model, shape, cfg, x_type, c_type, total, logs: List[int], stochastic, seeded, capture):
        dev = cfg.c_full.device
        nb = 2 * shape[0] if cfg.use_cfg else shape[0]
        self.x = torch.zeros(shape, device=dev, dtype=torch.float32)
        self.d_prev = torch.zeros_like(self.x)
        self.out = self.latent = torch.zeros(shape, device=dev, dtype=torch.float16)
        self.xin = torch.zeros((nb,) + tuple(shape[1:]), device=dev, dtype=torch.float16)
        super().__init__(model, shape, cfg, x_type, c_type, total, logs, stochastic, seeded, None, capture)

    def _one_step(self):
        # device-side loop header (step += 1, t = t(sigma_step)) -> UNet (+ControlNet) on the fp16 input x*c_in that
        # the previous update wrote into both CFG halves -> fused CFG combine + update (+ next input, output, logs)
        nv.ksampler_begin_step(self.step_idx, self.ttab, self.t_in)
        self.x_info["x"] = self.xin
        eps = self.model.apply_model(self.x_info, self.t_in, self.c_info)
        if self.device_noise:                      # stream 1, draw = the step index the header just advanced to
            rng.randn_into(self.noise, self.seeds, rng.STEP, 0, self.step_idx)
        nv.ksampler_step(eps, self.use_cfg, self.guidance, self.coef, self.step_idx, self.total - 1, self.x,
                         self.d_prev, self.xin, self.out, noise=self.noise if self.stochastic else None,
                         log_tab=self.log_tab, log_xt=self.log_xt, log_x0=self.log_x0)

    def load_request(self, xt, sigma0, cin0, c_full, cc, coef, ttab, seeds=None):
        self.x.copy_(xt)
        self.x.mul_(sigma0)                                              # sampler.py:89
        self.d_prev.zero_()
        b = self.x.shape[0]
        self.xin[:b].copy_(self.x * cin0)
        if self.use_cfg:
            self.xin[b:].copy_(self.xin[:b])
        self.step_idx.fill_(-1)
        super().load_request(c_full, cc, coef, ttab, seeds)
