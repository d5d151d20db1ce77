"""Float64 oracle for the k-diffusion samplers  —  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, in float64 torch on the CPU, what pfd_b200/sampler.py computes on the host and on the device:
  - the sigma schedule of the reference's Sampler.get_sigmas(n) (lib/model_zoo/sampler.py:29-54);
  - sigma_to_t, the inverse log-sigma interpolation (k-diffusion's DiscreteSchedule.sigma_to_t);
  - the per-step coefficient rows {sigma, a, b, c, u, c_in_next} of x' = a*x + b*D + c*D_prev + u*noise;
  - plain k-diffusion-style loops (Euler ancestral as sampler.py:84-104, DPM-Solver++(2M)) over any denoiser
    callable D(x, sigma), and the same loop driven by a coefficient table.
Pinned to the unmodified reference by tools/make_golden_sampler.py (tests/golden/sampler_reference.npz).
Only tests/ may import it; the product (pfd_b200/) never does.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence

import torch

Denoiser = Callable[[torch.Tensor, float], torch.Tensor]


def log_sigmas(alphas_cumprod: torch.Tensor) -> torch.Tensor:
    """sampler.py:38-39.  The table is formed in the dtype of `alphas_cumprod` (as the reference does; fp16 after
    net.half()) and returned in float64."""
    ac = alphas_cumprod.detach().cpu()
    return (((1 - ac) / ac) ** 0.5).log().double()


def get_sigmas(alphas_cumprod: torch.Tensor, n: int) -> torch.Tensor:
    """sampler.py:41-54: sigma(t) = exp(lerp(log_sigmas, t)) at t = linspace(T-1, 0, n), then a zero (float64)."""
    ls = log_sigmas(alphas_cumprod)
    t = torch.linspace(len(ls) - 1, 0, n).double()             # the reference's fp32 grid
    lo, hi = t.floor().long(), t.ceil().long()
    w = t - t.floor()
    return torch.cat([((1 - w) * ls[lo] + w * ls[hi]).exp(), torch.zeros(1, dtype=torch.float64)])


def sigma_to_t(sigma: torch.Tensor, ls: torch.Tensor) -> torch.Tensor:
    """k-diffusion DiscreteSchedule.sigma_to_t (float64)."""
    lsig = sigma.double().log()
    dists = lsig - ls[:, None]
    low = dists.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=ls.shape[0] - 2)
    high = low + 1
    lo, hi = ls[low], ls[high]
    w = torch.where(lo == hi, torch.zeros_like(lsig), (lo - lsig) / (lo - hi)).clamp(0, 1)
    return (1 - w) * low + w * high


def ancestral_step(sigma_from: float, sigma_to: float, eta: float = 1.0):
    """sampler.py:19-24."""
    if not eta:
        return sigma_to, 0.0
    up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    return (sigma_to ** 2 - up ** 2) ** 0.5, up


def coef_table(kind: str, sigmas: Sequence[float], eta: float = 1.0) -> torch.Tensor:
    """[steps, 6] float64 rows {sigma, a, b, c, u, c_in_next}."""
    s = [float(v) for v in sigmas]
    rows = []
    for i in range(len(s) - 1):
        sig, nxt = s[i], s[i + 1]
        if kind == "euler_a":
            # x + d*dt with d = (x - D)/sigma, dt = sigma_down - sigma   (sampler.py:98-101)
            down, up = ancestral_step(sig, nxt, eta)
            dt = down - sig
            a, b, c, u = 1 + dt / sig, -dt / sig, 0.0, up if nxt > 0 else 0.0
        elif kind == "dpmpp_2m":
            # t = -log(sigma); x' = (sigma'/sigma) x - expm1(-h) D', D' = (1 + 1/2r) D - (1/2r) D_prev on later steps
            if nxt == 0:
                a, b, c = 0.0, 1.0, 0.0
            else:
                h = -math.log(nxt) + math.log(sig)
                a, phi = nxt / sig, -math.expm1(-h)
                if i == 0:
                    b, c = phi, 0.0
                else:
                    r = (math.log(s[i - 1]) - math.log(sig)) / h
                    b, c = phi * (1 + 1 / (2 * r)), -phi / (2 * r)
            u = 0.0
        else:
            raise ValueError(kind)
        rows.append([sig, a, b, c, u, 1 / math.sqrt(nxt ** 2 + 1)])
    return torch.tensor(rows, dtype=torch.float64).reshape(-1, 6)


def run_table(denoise: Denoiser, x: torch.Tensor, table: torch.Tensor,
              noises: Optional[Sequence[torch.Tensor]] = None, trace: Optional[List] = None) -> torch.Tensor:
    """x_{i+1} = a x_i + b D_i + c D_{i-1} + u noise_i with D_i = denoise(x_i, sigma_i); noises[i] is the draw of step i
    (used where u != 0).  trace collects (x_i, D_i) per evaluation."""
    x = x.double()
    d_prev = torch.zeros_like(x)
    for i, (sig, a, b, c, u, _) in enumerate(table.tolist()):
        d = denoise(x, sig).double()
        if trace is not None:
            trace.append((x.clone(), d.clone()))
        xn = a * x + b * d + c * d_prev
        if u != 0.0:
            xn = xn + u * noises[i].double()
        x, d_prev = xn, d
    return x


def sample_euler_ancestral(denoise: Denoiser, x: torch.Tensor, sigmas: Sequence[float], eta: float = 1.0,
                           noises: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """sampler.py:84-104 in float64 (noises[i]: the randn_like draw of step i, sigma_{i+1} > 0)."""
    x = x.double()
    s = [float(v) for v in sigmas]
    for i in range(len(s) - 1):
        d = denoise(x, s[i]).double()
        down, up = ancestral_step(s[i], s[i + 1], eta)
        x = x + (x - d) / s[i] * (down - s[i])
        if s[i + 1] > 0 and up:
            x = x + noises[i].double() * up
    return x


def sample_dpmpp_2m(denoise: Denoiser, x: torch.Tensor, sigmas: Sequence[float]) -> torch.Tensor:
    """k-diffusion sample_dpmpp_2m in float64."""
    x = x.double()
    s = [float(v) for v in sigmas]
    old = None
    for i in range(len(s) - 1):
        d = denoise(x, s[i]).double()
        if s[i + 1] == 0:
            x = d
        else:
            t, tn = -math.log(s[i]), -math.log(s[i + 1])
            h = tn - t
            if old is None:
                dd = d
            else:
                r = (t + math.log(s[i - 1])) / h
                dd = (1 + 1 / (2 * r)) * d - (1 / (2 * r)) * old
            x = (s[i + 1] / s[i]) * x - math.expm1(-h) * dd
        old = d
    return x


def gaussian_denoiser(mu: torch.Tensor, s: float) -> Denoiser:
    """The exact denoiser E[x0 | x] for data x0 ~ N(mu, s^2) (elementwise): D = (s^2 x + sigma^2 mu) / (s^2 + sigma^2)."""
    return lambda x, sigma: (s * s * x + sigma * sigma * mu.to(x.dtype)) / (s * s + sigma * sigma)


def gaussian_ode_solution(mu: torch.Tensor, s: float, x_T: torch.Tensor, sigma_T: float, sigma: float):
    """Probability-flow ODE solution from (x_T, sigma_T) for N(mu, s^2) data:
    x(sigma) = mu + (x_T - mu) * sqrt(s^2 + sigma^2) / sqrt(s^2 + sigma_T^2)."""
    mu, x_T = mu.double(), x_T.double()
    return mu + (x_T - mu) * math.sqrt(s * s + sigma * sigma) / math.sqrt(s * s + sigma_T * sigma_T)
