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
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import native as nv
from . import rng
from .graphs import capture as graph_capture, weights_signature

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

        device = model.device
        seeds = x_info.get("seeds", None)
        seeded = seeds is not None
        if seeded:
            seeds = rng.seeds_tensor(rng.parse_seeds(seeds, int(shape[0])), device)
        if x_info.get("xt", None) is not None:
            xt = x_info["xt"].to(device=device)
        elif seeded:
            xt = torch.empty(tuple(shape), device=device, dtype=torch.float16)
            rng.randn_into(xt, seeds, rng.X_T)
        else:
            xt = torch.randn(shape, device=device, dtype=model.get_dtype())     # sampler.py:73
        guidance = float(c_info["unconditional_guidance_scale"])
        cond = c_info["conditioning"]
        uncond = c_info.get("unconditional_conditioning", None)
        use_cfg = not (guidance == 1.0 or uncond is None)
        c_full = (torch.cat([uncond, cond]) if use_cfg else cond).to(torch.float16).contiguous()
        cc = c_info.get("control", None)
        logs = log_steps(total, log_every_t)

        key = (tuple(xt.shape), tuple(c_full.shape), use_cfg, guidance, c_info["type"], x_info["type"],
               None if cc is None else (tuple(cc.shape), cc.dtype), total, stochastic, seeded, tuple(logs),
               weights_signature(model))
        st = self._states.get(key) if self.use_cuda_graph else None
        if st is None:
            st = _KSamplerState(model, tuple(xt.shape), c_full, cc, use_cfg, guidance, x_info["type"], c_info["type"],
                                total, stochastic, logs, capture=self.use_cuda_graph, seeded=seeded)
            if self.use_cuda_graph:
                if len(self._states) >= 2:
                    self._states.pop(next(iter(self._states)))
                self._states[key] = st
        st.load_request(xt, float(sig[0]), 1.0 / math.sqrt(sig[0] ** 2 + 1.0), c_full, cc,
                        torch.as_tensor(coef, dtype=torch.float32), torch.as_tensor(ts, dtype=torch.float32), seeds)
        st.run(sig)
        intermediates = {"pred_xt": [st.log_xt[s].clone() for s in range(len(logs))],
                         "pred_x0": [st.log_x0[s].clone() for s in range(len(logs))]}
        out = st.out.clone()
        x_info["x"] = out
        c_info["c"] = c_full
        return out, intermediates


class _KSamplerState:
    """Static buffers + captured graphs of one sampling configuration."""

    def __init__(self, model, shape, c_full, cc, use_cfg, guidance, x_type, c_type, total, stochastic,
                 logs: List[int], capture, seeded=False):
        dev = c_full.device
        self.model, self.use_cfg, self.guidance = model, use_cfg, guidance
        self.total, self.stochastic = total, stochastic
        # device-drawn noise (per-sample seeds): the loop needs no host work between steps
        self.device_noise = stochastic and seeded
        self.host_noise = stochastic and not seeded
        self.seeds = torch.zeros((shape[0],), device=dev, dtype=torch.int64)
        nb = 2 * shape[0] if use_cfg else shape[0]
        self.x = torch.zeros(shape, device=dev, dtype=torch.float32)
        self.d_prev = torch.zeros_like(self.x)
        self.out = torch.zeros(shape, device=dev, dtype=torch.float16)
        self.noise = torch.zeros(shape, device=dev, dtype=torch.float16)
        self.xin = torch.zeros((nb,) + tuple(shape[1:]), device=dev, dtype=torch.float16)
        self.c = torch.empty_like(c_full)
        self.cc = None if cc is None else torch.empty_like(cc)
        self.t_in = torch.zeros((nb,), device=dev, dtype=torch.float32)
        self.step_idx = torch.full((1,), -1, dtype=torch.int32, device=dev)
        self.coef = torch.zeros((total, nv.PFD_KSAMPLER_NCOEF), dtype=torch.float32, device=dev)
        self.ttab = torch.zeros((total,), dtype=torch.float32, device=dev)
        self.log_xt = torch.zeros((max(1, len(logs)),) + tuple(shape), device=dev, dtype=torch.float16)
        self.log_x0 = torch.zeros_like(self.log_xt)
        tab = torch.full((total,), -1, dtype=torch.int32)
        for slot, k in enumerate(logs):
            tab[k] = slot
        self.log_tab = tab.to(dev)
        self.x_info = {"type": x_type}
        self.c_info = {"type": c_type, "control": self.cc}
        self.prep_graph = self.step_graph = None
        self.n_prep = self.n_step = 0
        # eager pass first: builds every packed-weight cache and validates the launch sequence
        self.c.copy_(c_full)
        if cc is not None:
            self.cc.copy_(cc)
        self._prepare()
        if capture:
            self._one_step()                       # warm-up on scratch state (everything is re-loaded per request)
            torch.cuda.synchronize()
            self.prep_graph = torch.cuda.CUDAGraph()
            n0 = nv.launch_count()
            with graph_capture(self.prep_graph):
                self._prepare()
            self.n_prep = nv.launch_count() - n0
            self.step_graph = torch.cuda.CUDAGraph()
            n0 = nv.launch_count()
            with graph_capture(self.step_graph):
                for _ in range(1 if self.host_noise else total):
                    self._one_step()
            self.n_step = nv.launch_count() - n0

    def _prepare(self):
        prep = self.model.prepare_context(self.c, self.c_info["type"])
        if self.cc is not None and hasattr(self.model, "ctl"):
            prep["hint"] = self.model.ctl.hint_features(self.cc)
        self.c_info["c"] = prep["c"]
        self.c_info["_pfd_prepared"] = prep

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
        if seeds is not None:
            self.seeds.copy_(seeds)
        self.x.copy_(xt)
        self.x.mul_(sigma0)                                              # sampler.py:89
        self.d_prev.zero_()
        b = self.x.shape[0]
        self.xin[:b].copy_(self.x * cin0)
        if self.use_cfg:
            self.xin[b:].copy_(self.xin[:b])
        self.c.copy_(c_full)
        if cc is not None:
            self.cc.copy_(cc)
        self.coef.copy_(coef, non_blocking=True)
        self.ttab.copy_(ttab, non_blocking=True)
        self.step_idx.fill_(-1)
        if self.prep_graph is not None:
            self.prep_graph.replay()
            nv.note_replay(self.n_prep)
        else:
            self._prepare()

    def _step(self):
        if self.step_graph is not None:
            self.step_graph.replay()
            nv.note_replay(self.n_step)
        else:
            self._one_step()

    def run(self, sigmas):
        if not self.host_noise:
            if self.step_graph is not None:
                self._step()
            else:
                for _ in range(self.total):
                    self._one_step()
            return
        for i in range(self.total):
            if sigmas[i + 1] > 0:
                # sampler.py:102-103: one randn_like(x) per step with sigma_next > 0 (x is in the net's dtype);
                # normal_ on the static buffer draws the same values from the same generator
                self.noise.normal_()
            self._step()
