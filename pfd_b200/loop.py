"""The sampling loop shared by DDIMSampler (ddim.py) and the k-diffusion Sampler (sampler.py).

A LoopState holds the static device buffers of one sampling configuration and the CUDA graphs captured over them: a
prep graph (the step-invariant context K/V and hint stem) and a step graph of `spg` steps.  Each step is a device-side
loop header (step counter + timestep), the UNet (+ControlNet) and one fused update kernel.  A loop runs
  - eagerly (use_cuda_graph=False);
  - as a graph of spg steps replayed total / spg times (spg = the whole loop unless DDIM's steps_per_graph says less);
  - as a one-step graph per step, with torch's generator drawing the noise into the static `noise` buffer on the host
    before each step that adds noise: a stochastic loop without per-sample seeds.  With seeds (x_info["seeds"],
    rng.py) the noise is drawn on the device inside the graph, so the whole loop is one graph.
The states are cached across requests, keyed on shapes + a signature of the weights their graphs baked in.
"""
from __future__ import annotations

from collections import namedtuple
from typing import List

import torch

from . import rng
from .graphs import CapturedGraph, weights_signature

MAX_STATES = 2                          # sampling configurations (and their graphs) a sampler keeps

# the CFG batch of a request: guidance scale, whether the UNet runs on the [uncond | cond] pair, the fp16 context
# [uncond | cond] (or cond alone) and the ControlNet hint
Cfg = namedtuple("Cfg", "guidance use_cfg c_full cc")


def request_seeds(x_info, batch: int, device):
    """x_info["seeds"] as a [batch] int64 device tensor, or None for a request without per-sample seeds."""
    seeds = x_info.get("seeds", None)
    return None if seeds is None else rng.seeds_tensor(rng.parse_seeds(seeds, int(batch)), device)


def initial_noise(x_info, shape, seeds, device, dtype):
    """x_T: x_info["xt"], else drawn from the per-sample seeds (stream 0), else the reference's torch.randn in dtype."""
    if x_info.get("xt", None) is not None:
        return x_info["xt"].to(device=device)
    if seeds is not None:
        return rng.randn_into(torch.empty(tuple(shape), device=device, dtype=torch.float16), seeds, rng.X_T)
    return torch.randn(shape, device=device, dtype=dtype)


def cfg_context(c_info) -> Cfg:
    guidance = float(c_info["unconditional_guidance_scale"])
    cond = c_info["conditioning"]
    uncond = c_info.get("unconditional_conditioning", None)
    use_cfg = not (guidance == 1.0 or uncond is None)
    c_full = (torch.cat([uncond, cond]) if use_cfg else cond).to(torch.float16).contiguous()   # ddim.py:147
    return Cfg(guidance, use_cfg, c_full, c_info.get("control", None))


def state_key(model, x, cfg: Cfg, x_info, c_info, total: int, logs: List[int], *extra):
    cc = cfg.cc
    return (tuple(x.shape), tuple(cfg.c_full.shape), cfg.use_cfg, cfg.guidance, c_info["type"], x_info["type"],
            None if cc is None else (tuple(cc.shape), cc.dtype), total, tuple(logs)) + extra + (weights_signature(model),)


def cached_state(states: dict, key, use_cuda_graph: bool, build):
    """The state of `key`, built on a miss.  `states` keeps the MAX_STATES most recently built ones in insertion
    order; an eager sampler builds a fresh state per call and keeps none."""
    st = states.get(key) if use_cuda_graph else None
    if st is None:
        st = build()
        if use_cuda_graph:
            if len(states) >= MAX_STATES:
                states.pop(next(iter(states)))
            states[key] = st
    return st


class LoopState:
    """Static buffers + captured graphs of one sampling configuration.  A subclass allocates its own buffers (at least
    `latent`, the fp16 result) before calling __init__, and supplies _one_step() and load_request(), which loads the
    latent, resets the step counters and then calls LoopState.load_request."""

    T_DTYPE = None                      # dtype of the timestep table and the UNet's timestep input
    NCOEF = None                        # columns of the per-step coefficient table
    WARMUP_STEP = None                  # step counter before the warm-up step: its loop header lands on position 0

    def __init__(self, model, shape, cfg: Cfg, x_type, c_type, total: int, logs: List[int], stochastic: bool,
                 seeded: bool, steps_per_graph, capture: bool):
        dev = cfg.c_full.device
        self.model, self.use_cfg, self.guidance, self.total = model, cfg.use_cfg, cfg.guidance, total
        self.stochastic = stochastic
        self.device_noise = stochastic and seeded           # drawn inside the graph from the step counter
        self.host_noise = stochastic and not seeded         # drawn by torch's generator before each step
        if self.host_noise:
            self.spg = 1
        else:
            self.spg = max(1, min(steps_per_graph or total, total))
            while total % self.spg:
                self.spg -= 1
        nb = 2 * shape[0] if cfg.use_cfg else shape[0]
        self.seeds = torch.zeros((shape[0],), device=dev, dtype=torch.int64)
        self.noise = torch.zeros(shape, device=dev, dtype=torch.float16)
        self.c = torch.empty_like(cfg.c_full)
        self.cc = None if cfg.cc is None else torch.empty_like(cfg.cc)
        self.t_in = torch.zeros((nb,), device=dev, dtype=self.T_DTYPE)
        self.step_idx = torch.zeros(1, dtype=torch.int32, device=dev)
        self.coef = torch.zeros((total, self.NCOEF), dtype=torch.float32, device=dev)
        self.ttab = torch.zeros((total,), dtype=self.T_DTYPE, device=dev)
        self.n_logs = len(logs)
        self.log_xt = torch.zeros((max(1, len(logs)),) + tuple(shape), device=dev, dtype=torch.float16)
        self.log_x0 = torch.zeros_like(self.log_xt)
        tab = torch.full((total,), -1, dtype=torch.int32)
        for slot, k in enumerate(logs):
            tab[k] = slot
        self.log_tab = tab.to(dev)
        self.x_info = {"type": x_type}
        self.c_info = {"type": c_type, "control": self.cc}
        self.prep_graph = self.step_graph = None
        # eager pass first: builds every packed-weight cache and validates the launch sequence
        self.c.copy_(cfg.c_full)
        if cfg.cc is not None:
            self.cc.copy_(cfg.cc)
        self._prepare()
        if capture:
            self.step_idx.fill_(self.WARMUP_STEP)
            self._one_step()                   # warm-up on scratch state (everything is re-loaded per request)
            torch.cuda.synchronize()
            self.prep_graph = CapturedGraph(self._prepare)
            self.step_graph = CapturedGraph(self._steps)

    def _prepare(self):
        prep = self.model.prepare_context(self.c, self.c_info["type"])
        if self.cc is not None and hasattr(self.model, "ctl"):
            prep["hint"] = self.model.ctl.hint_features(self.cc)
        self.c_info["c"] = prep["c"]
        self.c_info["_pfd_prepared"] = prep

    def _steps(self):
        for _ in range(self.spg):
            self._one_step()

    def load_request(self, c_full, cc, coef, ttab, seeds=None):
        if seeds is not None:
            self.seeds.copy_(seeds)
        self.c.copy_(c_full)
        if cc is not None:
            self.cc.copy_(cc)
        self.coef.copy_(coef, non_blocking=True)
        self.ttab.copy_(ttab, non_blocking=True)
        if self.prep_graph is not None:
            self.prep_graph.replay()
        else:
            self._prepare()

    def run(self, draw_mask):
        """All steps of the loaded request.  draw_mask[i]: the host draws the noise of step i (host-noise loops)."""
        for i in range(0, self.total, self.spg):
            if self.host_noise and draw_mask[i]:
                # the reference loops' randn_like(x): the static fp16 buffer has x's shape, so this draws the same values
                # from the same generator, and a caller that substitutes torch.randn_like still feeds the update
                self.noise.copy_(torch.randn_like(self.noise))
            if self.step_graph is not None:
                self.step_graph.replay()
            else:
                self._steps()

    def result(self, x_info, c_info, c_full):
        """(fp16 latent, intermediates) of the finished loop; sets x_info["x"] and c_info["c"] like the reference."""
        intermediates = {"pred_xt": [self.log_xt[s].clone() for s in range(self.n_logs)],
                         "pred_x0": [self.log_x0[s].clone() for s in range(self.n_logs)]}
        out = self.latent.clone()
        x_info["x"] = out
        c_info["c"] = c_full
        return out, intermediates
