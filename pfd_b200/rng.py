"""Per-sample seeds: on-device counter-based Gaussian noise (pfd_randn_f16, include/pfd_b200.h).

A request opts in with x_info["seeds"]; every random draw of that request then comes from the sample's own seed:

    stream 0 (X_T):     the initial latent x_T
    stream 1 (STEP):    the sampler's per-step noise, draw index = schedule position k (0-based, in the order the
                        steps run), read from the device-side step counter inside the captured loop
    stream 2 (Q_SAMPLE): img2img's forward noise of x0

so "seed s" gives the same image whatever the batch size, the sample's position in it or the number of GPUs.
"""
from __future__ import annotations

import numbers
from typing import Optional, Sequence

import numpy as np
import torch

from . import native as nv

X_T, STEP, Q_SAMPLE = 0, 1, 2
_U64 = 1 << 64


def parse_seeds(seeds, batch: int) -> np.ndarray:
    """x_info["seeds"] -> uint64 array of `batch` seeds.  An int s means [s, s+1, ..., s+batch-1]; a sequence of ints or
    an integer tensor gives one seed per sample.  ValueError for a wrong length or a seed outside [0, 2^64)."""
    if isinstance(seeds, bool) or isinstance(seeds, np.bool_):
        raise ValueError("seeds: expected an int, a list of ints or an int64 tensor, got a bool")
    if isinstance(seeds, numbers.Integral):
        first = int(seeds)
        vals = [first + i for i in range(batch)]
    elif torch.is_tensor(seeds):
        if seeds.dtype.is_floating_point or seeds.dtype.is_complex or seeds.dtype == torch.bool or seeds.dim() != 1:
            raise ValueError(f"seeds: expected a 1-d integer tensor, got {seeds.dtype} of shape {tuple(seeds.shape)}")
        vals = [int(v) for v in seeds.detach().cpu().tolist()]
    elif isinstance(seeds, (list, tuple, np.ndarray)):
        vals = []
        for v in (seeds.tolist() if isinstance(seeds, np.ndarray) else seeds):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"seeds: {v!r} is not an int")
            vals.append(int(v))
    else:
        raise ValueError(f"seeds: expected an int, a list of ints or an int64 tensor, got {type(seeds).__name__}")
    if len(vals) != batch:
        raise ValueError(f"seeds: {len(vals)} seeds for a batch of {batch}")
    bad = [v for v in vals if not 0 <= v < _U64]
    if bad:
        raise ValueError(f"seeds: {bad[0]} is outside [0, 2^64)")
    return np.asarray(vals, dtype=np.uint64)


def seeds_tensor(seeds: np.ndarray, device) -> torch.Tensor:
    """uint64 seeds -> int64 tensor on `device` with the same bits (the layout pfd_randn_f16 reads)."""
    return torch.from_numpy(np.ascontiguousarray(seeds, dtype=np.uint64).view(np.int64).copy()).to(device)


def randn(shape: Sequence[int], seeds, stream: int = X_T, draw: int = 0, device=None) -> torch.Tensor:
    """fp16 N(0, 1) noise of `shape` [B, ...], sample b drawn from seed b: exactly what the samplers draw for a seeded
    request (stream 0 = x_T, 1 = per-step noise at schedule position `draw`, 2 = img2img forward noise).  `seeds` takes
    every form x_info["seeds"] does; device defaults to the current CUDA device."""
    shape = tuple(int(s) for s in shape)
    if len(shape) < 1 or shape[0] < 1:
        raise ValueError(f"randn: shape {shape} has no batch dimension")
    device = torch.device("cuda") if device is None else torch.device(device)
    s = seeds_tensor(parse_seeds(seeds, shape[0]), device)
    out = torch.empty(shape, device=device, dtype=torch.float16)
    if out.numel():
        nv.randn_f16(out, s, stream, draw)
    return out


def randn_into(out: torch.Tensor, seeds_dev: torch.Tensor, stream: int, draw: int = 0,
               draw_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Fill the static buffer `out` from the device seeds (graph-capturable; draw_dev = a device step counter)."""
    return nv.randn_f16(out, seeds_dev, stream, draw, draw_dev)
