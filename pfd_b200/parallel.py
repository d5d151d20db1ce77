"""Multi-GPU batch split for the sampler (SURVEY.md §8e): samples of a request are independent
inside the UNet / ControlNet / VAE (per-sample GroupNorm and attention; CFG pairs stay together), so
rank r simply takes samples [r*B/G, (r+1)*B/G).  No collective runs inside the 50-step loop; the
only exchanges are a broadcast of the conditioning at request start (or every rank re-encodes the
reference image) and a gather of the decoded images at the end.

Bit-parity with the single-GPU reference RNG stream (ddim.py:105) is kept by drawing the FULL
[B,4,L,L] noise with the reference seed on every rank and slicing.  A request with per-sample seeds
(x_info["seeds"], pfd_b200/rng.py) needs no such slice: each rank passes its own seeds (shard_seeds)
and draws only its own samples' noise.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(total: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced split of `total` samples; the first (total % world) ranks get one extra."""
    base, extra = divmod(total, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def sharded_noise(shape, seed: int, rank: int, world: int, device="cpu", dtype=torch.float32,
                  generator_device: Optional[str] = None) -> torch.Tensor:
    """x_T slice for this rank: full-batch randn with the request seed, then the rank's rows."""
    gdev = generator_device or device
    g = torch.Generator(device=gdev).manual_seed(seed)
    full = torch.randn(tuple(shape), generator=g, device=gdev, dtype=dtype)
    a, b = shard_range(shape[0], world, rank)
    return full[a:b].to(device)


def shard_seeds(seeds, world: int, rank: int) -> List[int]:
    """This rank's per-sample seeds: the shard_range slice of the request's full seed list (a list of ints, a
    numpy array or an integer tensor).  Every sample's noise depends only on its own seed, so the gathered
    images equal the single-GPU result."""
    if torch.is_tensor(seeds):
        vals = [int(v) for v in seeds.detach().cpu().tolist()]
    else:
        vals = [int(v) for v in seeds]
    a, b = shard_range(len(vals), world, rank)
    return vals[a:b]


def broadcast_conditioning(c: Optional[torch.Tensor], src: int = 0, shape=None, dtype=torch.float16,
                           device="cpu") -> torch.Tensor:
    """Broadcast the SeeCoder context (and any control map) from the rank that encoded it."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return c
    if dist.get_rank() != src:
        c = torch.empty(shape, dtype=dtype, device=device)
    dist.broadcast(c, src=src)
    return c


def gather_images(local: torch.Tensor, total: int) -> Optional[torch.Tensor]:
    """All-gather the decoded [b_r,3,H,W] images into the full [B,3,H,W] batch (ragged shards padded)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    per = max(shard_range(total, world, r)[1] - shard_range(total, world, r)[0] for r in range(world))
    pad = torch.zeros((per,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad)
    parts = []
    for r in range(world):
        a, b = shard_range(total, world, r)
        parts.append(bufs[r][: b - a])
    return torch.cat(parts, 0)
