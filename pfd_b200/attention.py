"""Multi-head attention on the C-ABI kernels (token-major fp16 tensors).

``project_heads`` runs the q/k/v projection GEMM whose epilogue scatters straight into the per-head
layouts the score/PV GEMMs consume (no transpose kernels):
    q, k : [B*heads, N, d]          (d contiguous = K-major operand of Q K^T)
    v^T  : [B*heads, d, Npad]       (keys contiguous = K-major B operand of P V)
``attend`` = batched Q K^T -> fp16 scores -> row softmax (reference rounding points, optional
relative-position bias / shift mask) -> batched P V written back as [B, Nq, heads*d].

Reference call sites: attention.py:178-201 (UNet/ControlNet CrossAttention), swin.py:179-210
(WindowAttention), seecoder.py:111,161 (nn.MultiheadAttention), autokl_modules.py:178-202.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import native as nv


# fused wgmma flash attention for bias-free attention; False falls back to the materialised
# QK^T GEMM -> softmax -> PV GEMM pipeline (still all pfd_b200 kernels) — used by tests to cross-check.
USE_FLASH = True
# fused q|k projection + V^T produced by a "swapped" GEMM (Wv . X^T), consumed by the v1 kernel through strided views
USE_FUSED_QK = True


def ceil8(n: int) -> int:
    return (n + 7) // 8 * 8


def project_heads(x2d: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], B: int, N: int,
                  heads: int, d: int, *, transposed: bool = False, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x2d [B*N, Cin] @ w[heads*d, Cin]^T (+b) -> [B*heads, Np, d] (or [B*heads, d, Np] if transposed).
    Np = ceil8(N); pad rows/cols are zero."""
    Np = ceil8(N)
    dev = x2d.device
    alloc = torch.zeros if Np != N else torch.empty
    if transposed:
        out = alloc((B * heads, d, Np), device=dev, dtype=torch.float16)
        so = (heads * d * Np, 0, 0, 1, d * Np, Np)
    else:
        out = alloc((B * heads, Np, d), device=dev, dtype=torch.float16)
        so = (heads * Np * d, 0, 0, d, Np * d, 1)
    ld = x2d.stride(0)
    segs = [(x2d, 1, x2d.shape[1], (ld, ld * N, ld * N))]
    if x2 is not None:
        segs.append((x2, 1, x2.shape[1], (x2.stride(0), x2.stride(0) * N, x2.stride(0) * N)))
    nv.gemm_raw(segs, in_w=N, in_h=1, stride=1, W=N, H=1, NB=B, w=w, N=w.shape[0], K=w.stride(0), bias=b,
                out=out, so=so, ndiv=1, cdiv=d)
    return out


def attend(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, *, B: int, heads: int, Nq: int, Nk: int,
           scale: float, bias: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
           nwin: int = 1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q [BH, Nqp, d], k [BH, Nkp, d], vt [BH, d, Nkp] -> out [B, Nq, heads*d]."""
    BH, Nqp, d = q.shape
    Nkp = k.shape[1]
    dev = q.device
    if USE_FLASH and bias is None and mask is None and d <= 192:
        if out is None:
            out = torch.empty((B, Nq, heads * d), device=dev, dtype=torch.float16)
        return nv.flash_attn(q, k, vt, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale, out=out)
    alloc = torch.zeros if Nkp != Nk else torch.empty
    s = alloc((BH, Nq, Nkp), device=dev, dtype=torch.float16)
    # S = Q K^T  (rows beyond Nq are not computed: the A raster is Nq wide)
    nv.gemm_raw([(q, 1, d, (d, d * Nqp, d * Nqp))], in_w=Nq, in_h=1, stride=1, W=Nq, H=1, NB=BH, w=k,
                N=Nkp, K=d, b_batch_stride=Nkp * d, out=s, so=(Nq * Nkp, 0, 0, Nkp, 0, 1))
    nv.softmax_(_view_cols(s, Nk), scale, bias=bias, nheads=heads, mask=mask, nwin=nwin)
    C = heads * d
    if out is None:
        out = torch.empty((B, Nq, C), device=dev, dtype=torch.float16)
    # O = P V  -> [B, Nq, heads*d]
    nv.gemm_raw([(s, 1, Nkp, (Nkp, Nkp * Nq, Nkp * Nq))], in_w=Nq, in_h=1, stride=1, W=Nq, H=1, NB=BH, w=vt,
                N=d, K=Nkp, b_batch_stride=d * Nkp, out=out, so=(Nq * C, d, 0, C, 0, 1), ndiv=heads)
    return out


def _view_cols(s: torch.Tensor, cols: int) -> torch.Tensor:
    # as_strided view keeps the row pitch (stride(1)) while exposing only the valid columns
    return s.as_strided((s.shape[0], s.shape[1], cols), (s.stride(0), s.stride(1), 1))


def project_heads_fused(x2d: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], B: int, N: int,
                        heads: int, d: int, nsec: int) -> torch.Tensor:
    """ONE projection GEMM for `nsec` stacked projections (q|k|v or k|v): x2d [B*N, Cin] @ w[nsec*heads*d, Cin]^T
    -> [B, nsec*heads, Np, d] (virtual heads).  Section s of the result is out[:, s*heads:(s+1)*heads]."""
    Np = ceil8(N)
    vh = nsec * heads
    alloc = torch.zeros if Np != N else torch.empty
    out = alloc((B, vh, Np, d), device=x2d.device, dtype=torch.float16)
    ld = x2d.stride(0)
    nv.gemm_raw([(x2d, 1, x2d.shape[1], (ld, ld * N, ld * N))], in_w=N, in_h=1, stride=1, W=N, H=1, NB=B, w=w,
                N=w.shape[0], K=w.stride(0), bias=b, out=out, so=(vh * Np * d, 0, 0, d, Np * d, 1), ndiv=1, cdiv=d)
    return out


def project_vt_swapped(x2d: torch.Tensor, wv: torch.Tensor, B: int, N: int, heads: int, d: int) -> torch.Tensor:
    """V^T for all batches with ONE vector-store GEMM: out[C, B*N] = Wv[C, Cin] @ x2d[B*N, Cin]^T (the weight is the
    A operand, the tokens are the K-major B operand).  Returns the strided view [B, heads, d, N]."""
    C, Cin = wv.shape
    T = x2d.shape[0]                                   # B*N tokens (N % 8 == 0 for the UNet self-attention)
    out = torch.empty((C, T), device=x2d.device, dtype=torch.float16)
    nv.gemm_raw([(wv, 1, Cin, (wv.stride(0), wv.stride(0) * C, wv.stride(0) * C))], in_w=C, in_h=1, stride=1, W=C,
                H=1, NB=1, w=x2d, N=T, K=x2d.stride(0), out=out, so=(0, 0, 0, T, 0, 1))
    return out.as_strided((B, heads, d, N), (N, d * T, T, 1))
