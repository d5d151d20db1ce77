"""DDIM sampler — mirrors lib/model_zoo/ddim.py:9-299 (`DDIMSampler(net).sample(steps, shape, x_info,
c_info, eta, ...) -> (x, intermediates)`, `p_sample_ddim`, `sample_multicontext`), with the schedule
maths reproduced operation for operation on the host (including the fp16-rounded `alphas_cumprod`
after `net.half()`, SURVEY.md App. C #6) and the per-step CFG combine + x_{t-1} update (+ eta noise)
fused into one CUDA kernel that reproduces the reference's fp16 rounding sequence (pfd_ddim_step_f16).

The sampling loop itself lives on the device (loop.py): the step counter, the timestep table and the
coefficient table are device buffers (pfd_ddim_begin_step), so ONE captured CUDA graph holds all
steps of a request (eta == 0) and is replayed with a single launch (`steps_per_graph` /
PFD_SAMPLER_STEPS_PER_GRAPH split it into shorter graphs); the graph is cached across requests, keyed
on shapes + a signature of the weights it baked in.  With eta > 0 and no seeds, a one-step graph that
ends in the noisy update is replayed per step, with the reference's per-step randn_like noise drawn
on the host in between.  With per-sample seeds (x_info["seeds"], pfd_b200/rng.py) x_T (stream 0),
img2img's forward noise (stream 2) and, for eta > 0, every step's noise (stream 1, drawn on the
device inside the graph) come from each sample's own seed, so the eta > 0 loop is one graph as well.
"""
from __future__ import annotations

import os
from typing import List

import numpy as np
import torch

from . import loop
from . import native as nv
from . import rng


def eta_is_zero(sigmas) -> bool:
    return not np.any(np.asarray(sigmas, dtype=np.float64) != 0.0)


def make_ddim_timesteps(num_ddim_timesteps, num_ddpm_timesteps):
    """diffusion_utils.py:32-46, 'uniform': stride T//S then +1 (steps=30 yields 31 evaluations)."""
    c = num_ddpm_timesteps // num_ddim_timesteps
    return np.asarray(list(range(0, num_ddpm_timesteps, c))) + 1


def _f16_round(values) -> torch.Tensor:
    """torch.full(shape, v, dtype=float16) rounding of python / numpy / 0-dim tensor scalars (ddim.py:160-163)."""
    if torch.is_tensor(values):
        return values.detach().cpu().to(torch.float16).to(torch.float32)
    return torch.as_tensor(np.asarray(values, dtype=np.float64)).to(torch.float16).to(torch.float32)


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.use_cuda_graph = kwargs.get("use_cuda_graph", True)
        # DDIM steps held by one captured graph: None = the whole loop (eta == 0)
        spg = kwargs.get("steps_per_graph", os.environ.get("PFD_SAMPLER_STEPS_PER_GRAPH"))
        self.steps_per_graph = int(spg) if spg else None
        self._states = {}

    def register_buffer(self, name, attr):
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0.0, verbose=True):
        """ddim.py:23-56 — same host ops in the same order."""
        if ddim_discretize != "uniform":
            raise NotImplementedError("only the 'uniform' DDIM discretisation is used by app.py")
        self.ddim_timesteps = make_ddim_timesteps(ddim_num_steps, self.ddpm_num_timesteps)
        ac = self.model.alphas_cumprod
        assert ac.shape[0] == self.ddpm_num_timesteps
        to32 = lambda x: x.clone().detach().to(torch.float32).cpu()
        self.betas = to32(self.model.betas)
        self.alphas_cumprod = to32(ac)
        self.alphas_cumprod_prev = to32(self.model.alphas_cumprod_prev)
        acc = self.alphas_cumprod
        ts = self.ddim_timesteps
        alphas = acc[ts]                                                 # fp32 torch tensor
        alphas_prev = np.asarray([acc[0]] + acc[ts[:-1]].tolist())       # float64 numpy (ddim.py via diffusion_utils:51)
        sigmas = ddim_eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
        self.ddim_sigmas, self.ddim_alphas, self.ddim_alphas_prev = sigmas, alphas, alphas_prev
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1.0 - alphas)
        # ddim.py:52-56 (use_original_steps=True path of p_sample_ddim)
        acf, acp = acc.double().numpy(), self.alphas_cumprod_prev.double().numpy()
        self.ddim_sigmas_for_original_num_steps = ddim_eta * np.sqrt((1 - acp) / (1 - acf) * (1 - acf / acp))

    def _coef_table(self, device=None) -> torch.Tensor:
        """[steps, 4] fp32 table {a_t, a_prev, sigma_t, sqrt(1-a_t)} of the per-step coefficients already
        rounded to fp16 the way torch.full(..., dtype=float16) rounds them (ddim.py:160-163)."""
        cols = [_f16_round(self.ddim_alphas), _f16_round(self.ddim_alphas_prev), _f16_round(self.ddim_sigmas),
                _f16_round(self.ddim_sqrt_one_minus_alphas)]
        tab = torch.stack(cols, 1).contiguous()
        return tab if device is None else tab.to(device)

    def _coef_original(self, index: int) -> torch.Tensor:
        m = self.model
        vals = [float(m.alphas_cumprod[index]), float(m.alphas_cumprod_prev[index]),
                float(self.ddim_sigmas_for_original_num_steps[index]), float(m.sqrt_one_minus_alphas_cumprod[index])]
        return _f16_round(vals).reshape(1, 4)

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sample(self, steps, shape, x_info, c_info, eta=0.0, temperature=1.0, noise_dropout=0.0, verbose=True,
               log_every_t=100):
        self.make_schedule(ddim_num_steps=steps, ddim_eta=eta, verbose=verbose)
        return self.ddim_sampling(shape, x_info=x_info, c_info=c_info, noise_dropout=noise_dropout,
                                  temperature=temperature, log_every_t=log_every_t)

    def _initial_latent(self, shape, x_info, dtype, timesteps, seeds=None):
        """ddim.py:94-105: returns (x_T fp16, timesteps actually walked).  seeds: per-sample device seeds (or None)."""
        model = self.model
        device = model.device
        if x_info.get("xt", None) is None and x_info.get("x0", None) is not None:
            # img2img branch (ddim.py:94-101): noise x0 forward to the n-th DDIM timestep (q_sample, pfd.py:204-207,
            # same torch.randn_like RNG call) and run only the first n timesteps of the schedule
            n_fwd = int(x_info["x0_forward_timesteps"])
            x0 = x_info["x0"].to(device=device, dtype=torch.float16).contiguous()
            t_fwd = int(timesteps[n_fwd])
            if seeds is not None:
                noise = rng.randn_into(torch.empty_like(x0), seeds, rng.Q_SAMPLE)
            else:
                noise = torch.randn_like(x0)
            x_T = nv.axpby(x0, float(model.sqrt_alphas_cumprod[t_fwd]), noise,
                           float(model.sqrt_one_minus_alphas_cumprod[t_fwd]))
            return x_T, timesteps[:n_fwd]
        # same RNG call as ddim.py:105 (dtype of the conditioning; fp16 on the GPU path)
        return loop.initial_noise(x_info, shape, seeds, device, dtype).to(torch.float16), timesteps

    @torch.no_grad()
    def ddim_sampling(self, shape, x_info, c_info, noise_dropout=0.0, temperature=1.0, log_every_t=100):
        """ddim.py:81-127.  The loop (per step: device-side step header -> CFG batch -> UNet [+ControlNet] ->
        fused CFG combine + DDIM update, in place on a static latent buffer) and the step-invariant
        preparation (cross-attention K/V of the context, ControlNet hint stem) are captured into CUDA
        graphs that are cached across calls, keyed on shapes + a signature of the weights they baked in."""
        model = self.model
        if noise_dropout > 0.0:
            raise NotImplementedError("noise_dropout is a training-time option not used by app.py")
        seeds = loop.request_seeds(x_info, shape[0], model.device)
        x_T, timesteps = self._initial_latent(shape, x_info, c_info["conditioning"].dtype, self.ddim_timesteps, seeds)
        cfg = loop.cfg_context(c_info)
        total = int(timesteps.shape[0])
        stochastic = not eta_is_zero(self.ddim_sigmas)
        seeded = seeds is not None
        log_idx = [i for i in range(total - 1, -1, -1) if i % log_every_t == 0 or i == total - 1]   # ddim.py:122
        # the update bakes temperature in whenever it adds noise
        key = loop.state_key(model, x_T, cfg, x_info, c_info, total, log_idx, stochastic, seeded,
                             self.steps_per_graph, float(temperature) if stochastic else None)
        st = loop.cached_state(self._states, key, self.use_cuda_graph, lambda: _DDIMState(
            model, x_T, cfg, x_info["type"], c_info["type"], total, log_idx, stochastic, seeded, self.steps_per_graph,
            self.use_cuda_graph, temperature))
        ttab = torch.as_tensor(np.ascontiguousarray(timesteps).astype(np.int64))
        st.load_request(x_T, cfg.c_full, cfg.cc, self._coef_table()[:total], ttab, seeds)
        st.run([True] * total)                                           # ddim.py:168 draws noise every step
        return st.result(x_info, c_info, cfg.c_full)

    # ------------------------------------------------------------------------------------------
    def _update(self, x, eps, guidance, index, use_original_steps, temperature, noise_dropout):
        """CFG combine + x_{t-1} update of one eagerly executed step (ddim.py:150-171)."""
        if noise_dropout > 0.0:
            raise NotImplementedError("noise_dropout is a training-time option not used by app.py")
        if use_original_steps:
            coef, sigma = self._coef_original(index).to(x.device), float(self.ddim_sigmas_for_original_num_steps[index])
            step = None
        else:
            coef, sigma = self._coef_table(x.device), float(self.ddim_sigmas[index])
            step = torch.tensor([index], dtype=torch.int32, device=x.device)
        x = x.to(torch.float16).contiguous()
        x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
        noise = torch.randn_like(x)                                      # ddim.py:168: drawn every step
        nv.ddim_step(eps, x, guidance, coef, step, x_prev, pred_x0, noise=noise if sigma != 0.0 else None,
                     temperature=temperature)
        return x_prev, pred_x0

    @torch.no_grad()
    def p_sample_ddim(self, x_info, c_info, t, index, repeat_noise=False, use_original_steps=False,
                      noise_dropout=0.0, temperature=1.0):
        """ddim.py:129-172: one (eager) DDIM step from x_info['x'] at timestep tensor t / schedule index."""
        if repeat_noise:
            raise NotImplementedError("repeat_noise is not used by the pfd pipelines")
        x = x_info["x"]
        guidance = float(c_info["unconditional_guidance_scale"])
        if guidance == 1.0 or c_info.get("unconditional_conditioning", None) is None:
            c_info["c"] = c_info["conditioning"]
            e = self.model.apply_model(x_info, t, c_info)
            eps = torch.cat([torch.zeros_like(e), e])                    # e_t = eps * scale (ddim.py:143-144)
        else:
            x_info["x"] = torch.cat([x] * 2)
            c_info["c"] = torch.cat([c_info["unconditional_conditioning"], c_info["conditioning"]])
            eps = self.model.apply_model(x_info, torch.cat([t] * 2), c_info)
        return self._update(x, eps, guidance, index, use_original_steps, temperature, noise_dropout)

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sample_multicontext(self, steps, shape, x_info, c_info_list, eta=0.0, temperature=1.0, noise_dropout=0.0,
                            verbose=True, log_every_t=100):
        """ddim.py:174-196."""
        self.make_schedule(ddim_num_steps=steps, ddim_eta=eta, verbose=verbose)
        return self.ddim_sampling_multicontext(shape, x_info=x_info, c_info_list=c_info_list,
                                               noise_dropout=noise_dropout, temperature=temperature,
                                               log_every_t=log_every_t)

    @torch.no_grad()
    def ddim_sampling_multicontext(self, shape, x_info, c_info_list, noise_dropout=0.0, temperature=1.0,
                                   log_every_t=100):
        """ddim.py:198-244 (eager: the mixed-context evaluation is adjacent functionality, SURVEY.md §8f)."""
        if x_info.get("seeds", None) is not None:
            raise NotImplementedError("x_info['seeds'] is supported by sample(), not by sample_multicontext()")
        bs = shape[0]
        x, timesteps = self._initial_latent(shape, x_info, c_info_list[0]["conditioning"].dtype, self.ddim_timesteps)
        x_info["x"] = x
        intermediates = {"pred_xt": [], "pred_x0": []}
        total = int(timesteps.shape[0])
        pred_xt = x
        for i, step in enumerate(np.flip(timesteps)):
            index = total - i - 1
            ts = torch.full((bs,), int(step), device=x.device, dtype=torch.long)
            pred_xt, pred_x0 = self.p_sample_ddim_multicontext(x_info, c_info_list, ts, index,
                                                               noise_dropout=noise_dropout, temperature=temperature)
            x_info["x"] = pred_xt
            if index % log_every_t == 0 or index == total - 1:
                intermediates["pred_xt"].append(pred_xt)
                intermediates["pred_x0"].append(pred_x0)
        return pred_xt, intermediates

    @torch.no_grad()
    def p_sample_ddim_multicontext(self, x_info, c_info_list, t, index, repeat_noise=False,
                                   use_original_steps=False, noise_dropout=0.0, temperature=1.0):
        """ddim.py:246-299."""
        if repeat_noise:
            raise NotImplementedError("repeat_noise is not used by the pfd pipelines")
        x = x_info["x"]
        guidance = None
        for c_info in c_info_list:
            if guidance is None:
                guidance = float(c_info["unconditional_guidance_scale"])
            else:
                assert guidance == float(c_info["unconditional_guidance_scale"]), \
                    "A different unconditional guidance scale between different context is not allowed!"
            if guidance == 1.0:
                c_info["c"] = c_info["conditioning"]
            else:
                c_info["c"] = torch.cat([c_info["unconditional_conditioning"], c_info["conditioning"]])
        if guidance == 1.0:
            e = self.model.apply_model_multicontext(x_info, t, c_info_list)
            eps = torch.cat([torch.zeros_like(e), e])
        else:
            x_info["x"] = torch.cat([x] * 2)
            eps = self.model.apply_model_multicontext(x_info, torch.cat([t] * 2), c_info_list)
        return self._update(x, eps, guidance, index, use_original_steps, temperature, noise_dropout)


class _DDIMState(loop.LoopState):
    """fp16 latent updated in place; the step counter counts down the schedule index (total-1, ..., 0)."""

    T_DTYPE, NCOEF, WARMUP_STEP = torch.long, 4, 1

    def __init__(self, model, x_T, cfg, x_type, c_type, total, log_idx: List[int], stochastic, seeded,
                 steps_per_graph, capture, temperature):
        self.temperature = float(temperature)
        self.x = self.latent = torch.zeros_like(x_T)
        self.pred_x0 = torch.zeros_like(x_T)
        if stochastic and seeded:
            # the draw index is the schedule position k = 0, 1, ... in the order the steps run, while the DDIM step
            # counter counts down: a second, ascending device counter advanced by the k-sampler's loop header (which
            # also writes the float k, unused, to k_t) holds k
            self.k_idx = torch.full((1,), -1, dtype=torch.int32, device=x_T.device)
            self.k_tab = torch.arange(total, dtype=torch.float32, device=x_T.device)
            self.k_t = torch.zeros((1,), dtype=torch.float32, device=x_T.device)
        super().__init__(model, tuple(x_T.shape), cfg, x_type, c_type, total, log_idx, stochastic, seeded,
                         steps_per_graph, capture)

    def _one_step(self):
        # device-side loop header (index -= 1, t = timesteps[index]; ddim.py:111-113) -> CFG batch (ddim.py:145-150)
        # -> UNet (+ControlNet) -> fused CFG combine + DDIM update (+ noise), in place on x
        nv.ddim_begin_step(self.step_idx, self.ttab, self.t_in)
        x = self.x
        self.x_info["x"] = torch.cat([x, x]) if self.use_cfg else x
        eps = self.model.apply_model(self.x_info, self.t_in, self.c_info)
        if not self.use_cfg:                                             # e_t = eps * scale (ddim.py:143-144)
            eps = torch.cat([torch.zeros_like(eps), eps])
        if self.device_noise:
            nv.ksampler_begin_step(self.k_idx, self.k_tab, self.k_t)
            rng.randn_into(self.noise, self.seeds, rng.STEP, 0, self.k_idx)
        nv.ddim_step(eps, x, self.guidance, self.coef, self.step_idx, x, self.pred_x0,
                     noise=self.noise if self.stochastic else None, temperature=self.temperature,
                     log_tab=self.log_tab, log_xt=self.log_xt, log_x0=self.log_x0)

    def load_request(self, x_T, c_full, cc, coef, ttab, seeds=None):
        self.x.copy_(x_T)
        self.step_idx.fill_(self.total)
        if self.device_noise:
            self.k_idx.fill_(-1)
        super().load_request(c_full, cc, coef, ttab, seeds)
