"""Parameter holders and weight packing shared by the pfd_b200 networks.

The networks keep the reference's module tree and parameter names (so ``load_state_dict(strict=True)``
of reference checkpoints works, app.py:137-162) by re-using torch.nn parameter containers — but their
``forward`` is disabled: all arithmetic goes through the C-ABI kernels in ``native`` on packed fp16
copies of the weights (channel-last / K-major layouts), built lazily and re-built whenever the
underlying parameter storage changes (load_state_dict, .half(), .to()).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .graphs import generation, watch


class _Holder:
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter holder: pfd_b200 computes through "
                           "the CUDA C-ABI kernels only (no torch fallback)")


class Conv2d(_Holder, nn.Conv2d):
    pass


class Linear(_Holder, nn.Linear):
    pass


class GroupNorm(_Holder, nn.GroupNorm):
    pass


class LayerNorm(_Holder, nn.LayerNorm):
    pass


class Embedding(_Holder, nn.Embedding):
    pass


class MultiheadAttention(_Holder, nn.MultiheadAttention):
    pass


class Container(nn.Module):
    """Plain attribute container (the reference uses bare nn.Module() for Decoder.mid / up levels)."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("container module")


class IndexedSequential(nn.Sequential):
    """Stands in for TimestepEmbedSequential / nn.Sequential: children keep their numeric names."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("pfd_b200 blocks are executed by their owner network")


# ------------------------------------------------------------------------------------------------
def cached(mod: nn.Module, key: str, params: Sequence[Optional[torch.Tensor]], fn: Callable):
    """Memoise fn() on `mod` until any tensor in `params` is replaced or modified in place."""
    store = mod.__dict__.get("_pfd_pk")
    if store is None:
        store = mod.__dict__.setdefault("_pfd_pk", {})
        watch(mod)
    sig = (generation(),) + tuple((p.data_ptr(), p._version, p.device.index) if p is not None else None
                                  for p in params)
    hit = store.get(key)
    if hit is None or hit[0] != sig:
        hit = (sig, fn())
        store[key] = hit
    return hit[1]


def fp16(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """A contiguous fp16 copy of a parameter (None stays None); the network must be on a CUDA device."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("pfd_b200 requires the network on a CUDA device (call net.to('cuda')); "
                           "there is no CPU execution path")
    return t.detach().to(torch.float16).contiguous()


def pad_rows(w: torch.Tensor, mult: int = 8) -> torch.Tensor:
    n = w.shape[0]
    if n % mult == 0:
        return w
    pad = torch.zeros((mult - n % mult,) + tuple(w.shape[1:]), device=w.device, dtype=w.dtype)
    return torch.cat([w, pad], 0).contiguous()


def pad_cols(w: torch.Tensor, mult: int = 8) -> torch.Tensor:
    k = w.shape[1]
    if k % mult == 0:
        return w
    pad = torch.zeros((w.shape[0], mult - k % mult), device=w.device, dtype=w.dtype)
    return torch.cat([w, pad], 1).contiguous()


def pack_conv(weight: torch.Tensor, cin: Optional[int] = None) -> torch.Tensor:
    """[O, I, k, k] -> fp16 [O, k*k*C] with K = tap*C + c (tap = ky*k + kx), the K order of pfd_gemm_f16; the input
    channels are zero-padded to C = cin when cin > I."""
    w = fp16(weight)
    o, i, kh, kw = w.shape
    if cin is not None and cin > i:
        w = torch.cat([w, w.new_zeros((o, cin - i, kh, kw))], 1)
    return w.permute(0, 2, 3, 1).reshape(o, -1).contiguous()


def pk_conv3(conv: nn.Conv2d, skip: Optional[nn.Conv2d] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Packed 3x3 weights (+ optional fused 1x1 skip conv appended along K, biases summed)."""
    def build():
        w = pack_conv(conv.weight)
        b = fp16(conv.bias)
        if skip is not None:
            ws = fp16(skip.weight).reshape(skip.weight.shape[0], -1)
            w = torch.cat([w, ws], 1).contiguous()
            if skip.bias is not None:
                b = (conv.bias.detach().float() + skip.bias.detach().float()).to(torch.float16).contiguous()
        if w.shape[0] % 8:
            w = pad_rows(w)
            b = pad_rows(b) if b is not None else None
        return w, b
    params = [conv.weight, conv.bias] + ([skip.weight, skip.bias] if skip is not None else [])
    return cached(conv, "conv3" + ("+skip" if skip is not None else ""), params, build)


def pk_conv3_small(conv: nn.Conv2d) -> Tuple[torch.Tensor, Optional[torch.Tensor], int]:
    """3x3 conv with tiny Cin (im2col path): weights [O, Kpad], Kpad = ceil8(9*Cin)."""
    def build():
        w = pad_cols(pack_conv(conv.weight))
        b = fp16(conv.bias)
        if w.shape[0] % 8:
            w, b = pad_rows(w), (pad_rows(b) if b is not None else None)
        return w, b, w.shape[1]
    return cached(conv, "conv3s", [conv.weight, conv.bias], build)


def pk_mat(mod: nn.Module, weight: torch.Tensor, bias: Optional[torch.Tensor], key: str = "mat",
           rows: Optional[slice] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Linear / 1x1-conv weights as [N, K] fp16 (optionally a row slice, e.g. one third of in_proj)."""
    def build():
        w = fp16(weight).reshape(weight.shape[0], -1)
        b = fp16(bias)
        if rows is not None:
            w = w[rows].contiguous()
            b = b[rows].contiguous() if b is not None else None
        if w.shape[1] % 8:
            w = pad_cols(w)
        if w.shape[0] % 8:
            w, b = pad_rows(w), (pad_rows(b) if b is not None else None)
        return w, b
    return cached(mod, key, [weight, bias], build)


def pk_lin(lin: nn.Module, key: str = "mat"):
    return pk_mat(lin, lin.weight, lin.bias, key)


def pk_norm(norm: nn.Module) -> Tuple[torch.Tensor, torch.Tensor]:
    return cached(norm, "norm", [norm.weight, norm.bias], lambda: (fp16(norm.weight), fp16(norm.bias)))


def pk_vec(mod: nn.Module, t: torch.Tensor, key: str) -> torch.Tensor:
    return cached(mod, key, [t], lambda: fp16(t))
