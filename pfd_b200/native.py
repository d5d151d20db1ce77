"""ctypes binding of the C-ABI kernel library (``libpfd_b200.so``, see ``include/pfd_b200.h``).

This is the *only* way compute reaches the GPU in this package: there is no torch / CPU fallback.
If the shared library is missing or a call fails, a ``RuntimeError`` is raised.

The argument and return types of every entry point come from its prototype in ``include/pfd_b200.h``.  Tensors go
into pointer arguments as they are (``DevicePtr``); the stream is torch's current stream so calls can be captured
into CUDA graphs.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_uint32, c_void_p
from typing import Dict, List, Optional, Sequence, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# PFD_B200_LIB: load another build of the same ABI (A/B runs of compile-time variants); default = the in-tree library
LIB_PATH = os.environ.get("PFD_B200_LIB") or os.path.join(_HERE, "libpfd_b200.so")
HEADER = os.path.join(_HERE, os.pardir, "include", "pfd_b200.h")

# mirrors of the header's #defines (tests/test_abi_cpu.py keeps them equal)
PFD_MAX_SEG = 3
ACT_NONE, ACT_SILU, ACT_GELU, ACT_RELU, ACT_GEGLU = 0, 1, 2, 3, 4
PFD_KSAMPLER_NCOEF = 6
PFD_HED_MAX_SIDES = 5
PFD_PIDINET_SIDE_PARAMS = 161
PFD_MLSD_TOPK = 200
PFD_OPENPOSE_MAX_PEAKS = 128
PFD_OPENPOSE_MAX_PERSONS = 17 * PFD_OPENPOSE_MAX_PEAKS


class GemmDesc(ctypes.Structure):
    """Mirror of ``pfd_gemm_desc`` (include/pfd_b200.h)."""
    _fields_ = [
        ("nseg", c_int32),
        ("taps", c_int32 * PFD_MAX_SEG),
        ("a_c", c_int32 * PFD_MAX_SEG),
        ("a_ptr", c_void_p * PFD_MAX_SEG),
        ("a_sx", c_int64 * PFD_MAX_SEG),
        ("a_sy", c_int64 * PFD_MAX_SEG),
        ("a_sn", c_int64 * PFD_MAX_SEG),
        ("in_w", c_int32), ("in_h", c_int32),
        ("stride", c_int32),
        ("W", c_int32), ("H", c_int32), ("NB", c_int32),
        ("b_ptr", c_void_p),
        ("N", c_int32),
        ("K", c_int64),
        ("b_batch_stride", c_int64),
        ("alpha", c_float),
        ("act", c_int32),
        ("bias", c_void_p),
        ("rowadd", c_void_p),
        ("rowadd_ld", c_int64),
        ("residual", c_void_p),
        ("out", c_void_p),
        ("so_n1", c_int64), ("so_n0", c_int64), ("so_y", c_int64), ("so_x", c_int64),
        ("so_c1", c_int64), ("so_c0", c_int64),
        ("ndiv", c_int32), ("cdiv", c_int32),
        ("bn_force", c_int32),
        ("tap_off", c_int32),
        ("stream", c_void_p),
    ]


class DevicePtr(c_void_p):
    """Type of every pointer argument: a CUDA tensor passes its data_ptr(), None passes NULL, and whatever c_void_p
    accepts (ints, ctypes arrays, byref) passes unchanged.  A tensor that is not on a CUDA device is refused before
    the call (ctypes.ArgumentError naming the argument's position) instead of reaching a kernel as a host address."""

    @classmethod
    def from_param(cls, obj):
        if isinstance(obj, torch.Tensor):
            if not obj.is_cuda:
                raise TypeError(f"expected a CUDA tensor, got a {obj.dtype} tensor on {obj.device}")
            obj = obj.data_ptr()
        return c_void_p.from_param(obj)


# C type of the header -> ctypes type; any other pointer type is a DevicePtr
_CTYPES = {"int": c_int32, "int32_t": c_int32, "uint32_t": c_uint32, "int64_t": c_int64, "float": c_float,
           "const char*": c_char_p, "const pfd_gemm_desc*": POINTER(GemmDesc)}


def _prototypes() -> Dict[str, Tuple[str, List[str]]]:
    """{name: (return type, [parameter types])} of every PFD_API prototype in HEADER, types with normalised spaces."""
    with open(HEADER) as f:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", "", f.read(), flags=re.S)
    norm = lambda t: re.sub(r"\s*\*", "*", " ".join(t.split()))
    protos = {}
    for ret, name, params in re.findall(r"PFD_API\s+([\w\s\*]+?)\s*\b(pfd_\w+)\s*\(([^)]*)\)", src):
        params = [] if params.strip() == "void" else [re.sub(r"\w+\s*$", "", p) for p in params.split(",")]
        protos[name] = (norm(ret), [norm(p) for p in params])
    return protos


def _ctype(name: str, t: str):
    if t in _CTYPES:
        return _CTYPES[t]
    if t.endswith("*"):
        return DevicePtr
    raise RuntimeError(f"{name}: the C type '{t}' of include/pfd_b200.h has no ctypes mapping in native._CTYPES")


EXPORTS = tuple(_prototypes())
_lib = None


def _declare(lib):
    """Set argtypes and restype of every function the header declares on lib; raises on a type without a mapping and
    on declared functions lib lacks."""
    protos = _prototypes()
    missing = [name for name in protos if not hasattr(lib, name)]
    if missing:
        raise RuntimeError(f"{LIB_PATH} lacks functions that include/pfd_b200.h declares: {', '.join(missing)}")
    for name, (ret, params) in protos.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = _ctype(name, ret), [_ctype(name, t) for t in params]
    return lib


def load() -> ctypes.CDLL:
    """Load the shared library (once) and declare its functions from the header.  Raises if it has not been built
    (``__graft_entry__.build``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU/PyTorch fallback for the pfd_b200 kernels)")
    _lib = _declare(ctypes.CDLL(LIB_PATH))
    return _lib


def _check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().pfd_last_error()
        raise RuntimeError(f"{what} failed: {msg.decode() if msg else rc}")


def env_flag(value: Optional[str]) -> bool:
    """Value of an on/off environment switch (PFD_DETERMINISTIC, PFD_NO_PDL): on when it starts with '1'."""
    return bool(value) and value[0] == "1"


# Deterministic mode (pfd_set_option "deterministic"): the library reads PFD_DETERMINISTIC once when it is loaded and
# uses it as the option's default; this mirror follows the option so Python can tell which mode is in effect.
_DETERMINISTIC_DEFAULT = env_flag(os.environ.get("PFD_DETERMINISTIC"))
_deterministic = _DETERMINISTIC_DEFAULT


def deterministic() -> bool:
    return _deterministic


def set_env_option(name: Optional[str], value) -> None:
    """Library tuning switch (pfd_set_option); name=None resets every switch to its default.  Setting "deterministic"
    here does not drop captured CUDA graphs; pfd_b200.set_deterministic() does."""
    global _deterministic
    _check(load().pfd_set_option(None if name is None else name.encode(), 0 if value is None else int(value)),
           "pfd_set_option")
    if name is None:
        _deterministic = _DETERMINISTIC_DEFAULT
    elif name == "deterministic":
        _deterministic = bool(int(value or 0))


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


_replayed = 0


def note_replay(n: int) -> None:
    """Account for kernels re-launched by a CUDA-graph replay (they bypass the library's counter)."""
    global _replayed
    _replayed += int(n)


def launch_count() -> int:
    """Kernels launched by this library in this process (direct launches + graph-replayed ones)."""
    return int(load().pfd_launch_count()) + _replayed


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    """Address of an optional tensor, for the pointer fields of GemmDesc (function arguments take tensors directly)."""
    if t is None:
        return None
    return t.data_ptr()


def _call(name: str, *args) -> None:
    """The library function `name` on (*args, current stream); raises RuntimeError with the library's error text when
    it fails.  The library is looked up on every call, so a test can replace load()."""
    _check(getattr(load(), name)(*args, stream_ptr()), name)


def _chk16(t: torch.Tensor, name: str) -> None:
    if t.dtype != torch.float16 or not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA fp16 tensor, got {t.dtype} on {t.device}")


def _chk32(t: torch.Tensor, name: str) -> None:
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise RuntimeError(f"{name}: expected a contiguous CUDA fp32 tensor, got {t.dtype} on {t.device}")


def _chk_image(x: torch.Tensor, what: str) -> Tuple[torch.Tensor, int]:
    """An NCHW [B,3,H,W] CUDA fp16/fp32 image -> (x contiguous, 1 if it is fp32 else 0)."""
    if x.dim() != 4 or x.shape[1] != 3 or not x.is_cuda or x.dtype not in (torch.float16, torch.float32):
        raise RuntimeError(f"{what}: expected a CUDA fp16/fp32 [B,3,H,W] image, got {tuple(x.shape)} {x.dtype} "
                           f"{x.device}")
    return x.contiguous(), int(x.dtype == torch.float32)


# --------------------------------------------------------------------------------------------
# GEMM family
# --------------------------------------------------------------------------------------------
def gemm_raw(segs: Sequence[Tuple[torch.Tensor, int, int, Tuple[int, int, int]]], *, in_w: int,
             in_h: int, stride: int, W: int, H: int, NB: int, w: torch.Tensor, N: int, K: int,
             b_batch_stride: int = 0, alpha: float = 1.0, act: int = ACT_NONE,
             bias: Optional[torch.Tensor] = None, rowadd: Optional[torch.Tensor] = None,
             residual: Optional[torch.Tensor] = None, out: torch.Tensor,
             so: Tuple[int, int, int, int, int, int], ndiv: int = 1, cdiv: int = 0,
             bn_force: int = 0, tap_off: int = 0) -> None:
    """Lowest-level call: ``segs`` is a list of (tensor, taps, channels, (sx, sy, sn))."""
    d = GemmDesc()
    d.nseg = len(segs)
    for i, (t, taps, c, (sx, sy, sn)) in enumerate(segs):
        _chk16(t, f"A[{i}]")
        d.taps[i] = taps
        d.a_c[i] = c
        d.a_ptr[i] = t.data_ptr()
        d.a_sx[i], d.a_sy[i], d.a_sn[i] = sx, sy, sn
    d.in_w, d.in_h, d.stride = in_w, in_h, stride
    d.W, d.H, d.NB = W, H, NB
    _chk16(w, "B")
    d.b_ptr = w.data_ptr()
    d.N, d.K, d.b_batch_stride = N, K, b_batch_stride
    d.alpha, d.act = alpha, act
    d.bias = _p(bias)
    d.rowadd = _p(rowadd)
    d.rowadd_ld = rowadd.stride(0) if rowadd is not None else 0
    d.residual = _p(residual)
    d.out = out.data_ptr()
    d.so_n1, d.so_n0, d.so_y, d.so_x, d.so_c1, d.so_c0 = so
    d.ndiv, d.cdiv = ndiv, cdiv
    d.bn_force = bn_force
    d.tap_off = tap_off
    d.stream = stream_ptr()
    _check(load().pfd_gemm_f16(ctypes.byref(d)), "pfd_gemm_f16")


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: int = ACT_NONE,
           residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
           alpha: float = 1.0, x2: Optional[torch.Tensor] = None, bn_force: int = 0) -> torch.Tensor:
    """out[M, N] = act(alpha * [x | x2] @ w^T + bias) + residual.  x: [M, K1] (row pitch = stride(0)),
    optional x2: [M, K2]; w: [N, K1+K2] (GEGLU: tile-packed, output has N/2 columns)."""
    M, K1 = x.shape
    N = w.shape[0]
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), device=x.device, dtype=torch.float16)
    segs = [(x, 1, K1, (x.stride(0), x.stride(0) * M, x.stride(0) * M))]
    if x2 is not None:
        segs.append((x2, 1, x2.shape[1], (x2.stride(0), x2.stride(0) * M, x2.stride(0) * M)))
    ldo = out.stride(0)
    gemm_raw(segs, in_w=M, in_h=1, stride=1, W=M, H=1, NB=1, w=w, N=N, K=w.stride(0), alpha=alpha,
             act=act, bias=bias, residual=residual, out=out, so=(0, 0, 0, ldo, 0, 1), bn_force=bn_force)
    return out


def geglu_tile(n2: int) -> int:
    """N-tile width used for a GEGLU projection with 2*inner = n2 output features."""
    for bn in (160, 256, 128, 192, 64):
        if n2 % bn == 0:
            return bn
    raise RuntimeError(f"GEGLU width {n2} is not divisible by any supported N tile")


def pack_geglu(w: torch.Tensor, b: Optional[torch.Tensor]):
    """Re-order GEGLU.proj rows (attention.py:47-51: first half = value, second half = gate) so every
    N tile holds [value(bn/2) | gate(bn/2)] for the same output columns. Returns (w, b, bn)."""
    n2 = w.shape[0]
    inner = n2 // 2
    bn = geglu_tile(n2)
    h = bn // 2
    idx = torch.arange(n2, device=w.device).reshape(n2 // bn, 2, h)
    tile = torch.arange(n2 // bn, device=w.device).reshape(-1, 1)
    j = torch.arange(h, device=w.device).reshape(1, -1)
    src = torch.stack([tile * h + j, inner + tile * h + j], dim=1).reshape(-1)
    wp = w.index_select(0, src).contiguous()
    bp = b.index_select(0, src).contiguous() if b is not None else None
    return wp, bp, bn


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, stride: int = 1,
            rowadd: Optional[torch.Tensor] = None, act: int = ACT_NONE,
            residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
            skip: Sequence[torch.Tensor] = (), tap_off: int = 0) -> torch.Tensor:
    """3x3 / pad 1 convolution on channel-last x [NB, H, W, C] with packed weights
    w [Cout, 9*C (+ sum of skip channels)] (k = tap*C + c, then the 1x1 skip-segment channels).
    ``skip`` tensors (same raster, stride 1 only) are extra 1x1 K-segments accumulated into the same
    output — used to fuse ResBlock.skip_connection(x) (openaimodel.py:240,274) into out_layers' conv."""
    NB, H, W, C = x.shape
    # padding (1 - tap_off) on the top/left, 1 on the bottom/right: tap_off = 1 is F.pad(x, (0,1,0,1)) + padding 0
    Ho, Wo = (H - 1 - tap_off) // stride + 1, (W - 1 - tap_off) // stride + 1
    N = w.shape[0]
    if out is None:
        out = torch.empty((NB, Ho, Wo, N), device=x.device, dtype=torch.float16)
    segs = [(x, 9, C, (x.stride(2), x.stride(1), x.stride(0)))]
    for s in skip:
        segs.append((s, 1, s.shape[3], (s.stride(2), s.stride(1), s.stride(0))))
    gemm_raw(segs, in_w=W, in_h=H, stride=stride, W=Wo, H=Ho, NB=NB, w=w, N=N, K=w.stride(0), act=act,
             bias=bias, rowadd=rowadd, residual=residual, out=out,
             so=(out.stride(0), 0, out.stride(1), out.stride(2), 0, 1), tap_off=tap_off)
    return out


def conv1x1(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: int = ACT_NONE,
            residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
            x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """1x1 conv on channel-last tensors == linear over flattened pixels."""
    NB, H, W, C = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((NB, H, W, N), device=x.device, dtype=torch.float16)
    r = residual.reshape(NB * H * W, -1) if residual is not None else None
    linear(x.reshape(NB * H * W, C), w, bias, act=act, residual=r, out=out.reshape(NB * H * W, N),
           x2=None if x2 is None else x2.reshape(NB * H * W, -1))
    return out


def conv1x1_into(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, *,
                 act: int = ACT_NONE) -> torch.Tensor:
    """act(1x1 conv of x + bias) between channel-last views: x [NB,H,W,C] and out [NB,H,W,N] may have any pixel
    strides (e.g. channel slices of concat buffers) but unit channel stride."""
    NB, H, W, C = x.shape
    gemm_raw([(x, 1, C, (x.stride(2), x.stride(1), x.stride(0)))], in_w=W, in_h=H, stride=1, W=W, H=H, NB=NB, w=w,
             N=w.shape[0], K=w.stride(0), act=act, bias=bias, out=out,
             so=(out.stride(0), 0, out.stride(1), out.stride(2), 0, 1))
    return out


def bmm_nt(a: torch.Tensor, b: torch.Tensor, *, out: torch.Tensor, so, ndiv: int = 1, cdiv: int = 0,
           alpha: float = 1.0) -> None:
    """Batched out[b] = a[b] @ b[b]^T.  a: [B, M, K] contiguous-in-K, b: [B, N, K]; generic out strides."""
    B, M, K = a.shape
    N = b.shape[1]
    gemm_raw([(a, 1, K, (a.stride(1), a.stride(1) * M, a.stride(0)))], in_w=M, in_h=1, stride=1, W=M,
             H=1, NB=B, w=b, N=N, K=b.stride(1), b_batch_stride=b.stride(0), alpha=alpha, out=out,
             so=so, ndiv=ndiv, cdiv=cdiv)


# --------------------------------------------------------------------------------------------
# normalisation / softmax / misc
# --------------------------------------------------------------------------------------------
# GroupNorm statistics scratch: a ring of pre-zeroed slots per (device, stream).  `gn_reset()` zeroes the
# whole ring with ONE memset (called at the start of every network evaluation); each groupnorm() call then
# takes the next slot without a memset of its own.  If the ring is exhausted the call zeroes a fallback slot itself.
# Deterministic mode uses the same slots: its per-chunk partials live in a library-owned per-device buffer, and only
# the final (sum, sumsq) per (image, group) is written to the slot, so neither the slot size nor the per-evaluation
# memset grows.
_GN_SLOT_BYTES = 64 * 32 * 16 + 256    # up to 64 images x 32 groups x (sum, sumsq) fp64 (+ spare)
_GN_SLOTS = 256
_gn_rings = {}


def _gn_ring():
    key = (torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    ring = _gn_rings.get(key)
    if ring is None:
        buf = torch.zeros(_GN_SLOT_BYTES * (_GN_SLOTS + 1), device="cuda", dtype=torch.uint8)   # + 1 fallback slot
        ring = {"buf": buf, "next": _GN_SLOTS}      # exhausted until the first gn_reset()
        _gn_rings[key] = ring
    return ring


def gn_reset() -> None:
    """Zero all GroupNorm scratch slots of the current stream (one memset) and rewind the ring."""
    ring = _gn_ring()
    ring["buf"].zero_()
    ring["next"] = 0


def groupnorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, *, silu: bool,
              x2: Optional[torch.Tensor] = None, groups: int = 32,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm(+SiLU) over channel-last x [NB, H, W, C1] (optionally concatenated with x2 [.., C2])."""
    NB, H, W, C1 = x.shape
    C2 = x2.shape[3] if x2 is not None else 0
    if out is None:
        out = torch.empty((NB, H, W, C1 + C2), device=x.device, dtype=torch.float16)
    ring = _gn_ring()
    need = NB * groups * 16 + NB * 4
    if ring["next"] < _GN_SLOTS and need <= _GN_SLOT_BYTES:
        ws_ptr, zero = ring["buf"].data_ptr() + ring["next"] * _GN_SLOT_BYTES, 0
        ring["next"] += 1
    else:
        if need > _GN_SLOT_BYTES:
            raise RuntimeError("groupnorm: batch too large for the statistics scratch")
        ws_ptr, zero = ring["buf"].data_ptr() + _GN_SLOTS * _GN_SLOT_BYTES, 1    # shared fallback slot, zeroed per call
        ring["next"] = _GN_SLOTS
    _call("pfd_groupnorm_f16", x, C1, x2, C2, NB, H * W, groups, gamma, beta, eps, int(silu), out, ws_ptr, zero)
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, *,
              residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _call("pfd_layernorm_f16", x, residual, rows, C, gamma, beta, eps, out)
    return out


def softmax_(s: torch.Tensor, scale: float, *, bias: Optional[torch.Tensor] = None, nheads: int = 1,
             mask: Optional[torch.Tensor] = None, nwin: int = 1) -> torch.Tensor:
    """In-place row softmax over s [batch, rows, cols] (see pfd_softmax_f16).  Rows may be padded (stride(1) >= cols)
    but the batches must be packed; bias is [nheads, rows, cols] (picked by b % nheads) and mask [nwin, rows, cols]
    (picked by (b / nheads) % nwin), both contiguous."""
    _chk16(s, "softmax_: s")
    if s.dim() != 3:
        raise ValueError(f"softmax_: s must be [batch, rows, cols], got {tuple(s.shape)}")
    batch, rows, cols = s.shape
    if s.stride(2) != 1 or s.stride(1) < cols or s.stride(0) != rows * s.stride(1):
        raise ValueError(f"softmax_: s {tuple(s.shape)} needs unit column stride, a row pitch >= cols and packed "
                         f"batches, got strides {s.stride()}")
    for t, n, name in ((bias, nheads, "bias"), (mask, nwin, "mask")):
        if t is not None:
            _chk16(t, f"softmax_: {name}")
            if tuple(t.shape) != (max(n, 1), rows, cols) or not t.is_contiguous():
                raise ValueError(f"softmax_: {name} must be a contiguous [{max(n, 1)}, {rows}, {cols}] tensor, "
                                 f"got {tuple(t.shape)} with strides {t.stride()}")
    _call("pfd_softmax_f16", s, batch, rows, cols, s.stride(1), scale, bias, nheads, mask, nwin)
    return s


def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """[cos | sin] embedding of int64 timesteps (the DDIM sampler) or float32 fractional ones (the k-samplers)."""
    out = torch.empty((t.shape[0], dim), device=t.device, dtype=torch.float16)
    if t.dtype == torch.int64:
        _call("pfd_timestep_embedding_f16", t, t.shape[0], dim, max_period, out)
    elif t.dtype == torch.float32:
        _call("pfd_timestep_embedding_ft_f16", t.contiguous(), t.shape[0], dim, max_period, out)
    else:
        raise RuntimeError(f"timestep_embedding: int64 or float32 timesteps expected, got {t.dtype}")
    return out


def upsample2x(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    NB, H, W, C = x.shape
    if out is None:
        out = torch.empty((NB, 2 * H, 2 * W, C), device=x.device, dtype=torch.float16)
    _call("pfd_upsample2x_f16", x, NB, H, W, C, out)
    return out


def nchw_to_nhwc(x: torch.Tensor, cpad: Optional[int] = None, out: Optional[torch.Tensor] = None, *,
                 mul: float = 1.0, add: float = 0.0) -> torch.Tensor:
    NB, C, H, W = x.shape
    cpad = cpad or C
    x = x.contiguous()
    if out is None:
        out = torch.empty((NB, H, W, cpad), device=x.device, dtype=torch.float16)
    if x.dtype not in (torch.float16, torch.float32):
        raise RuntimeError(f"nchw_to_nhwc: unsupported dtype {x.dtype}")
    _call("pfd_nchw_to_nhwc_f16", x, int(x.dtype == torch.float32), NB, C, H, W, cpad, mul, add, out)
    return out


def nhwc_to_nchw(x: torch.Tensor, C: Optional[int] = None, *, mul: float = 1.0, add: float = 0.0,
                 lo: float = -65504.0, hi: float = 65504.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    NB, H, W, Cpad = x.shape
    C = C or Cpad
    if out is None:
        out = torch.empty((NB, C, H, W), device=x.device, dtype=torch.float16)
    _call("pfd_nhwc_to_nchw_f16", x, NB, C, H, W, Cpad, mul, add, lo, hi, out)
    return out


def im2col3x3(x: torch.Tensor, kpad: int, stride: int = 1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    NB, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty((NB, Ho, Wo, kpad), device=x.device, dtype=torch.float16)
    _call("pfd_im2col3x3_f16", x, NB, H, W, C, stride, kpad, out)
    return out


def conv3x3_im2col(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor] = None, *, stride: int = 1,
                   act: int = ACT_NONE) -> torch.Tensor:
    """3x3 / pad 1 convolution of channel-last x [NB, H, W, C] whose C is too small for conv3x3's TMA path (UNet / VAE
    conv_in, the ControlNet hint stem, the annotators' RGB input): im2col3x3 to K = w.shape[1] columns, then linear.
    w: [N, K] packed as k = tap*C + c, zero columns up to K -> [NB, Ho, Wo, N]."""
    col = im2col3x3(x, w.shape[1], stride)
    NB, Ho, Wo, K = col.shape
    return linear(col.reshape(NB * Ho * Wo, K), w, b, act=act).reshape(NB, Ho, Wo, w.shape[0])


def axpby(a: torch.Tensor, sa: float, b: Optional[torch.Tensor] = None, sb: float = 0.0,
          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty_like(a)
    _call("pfd_axpby_f16", a, sa, b, sb, a.numel(), out)
    return out


def add_rowvec(a: torch.Tensor, row: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    C = a.shape[-1]
    if out is None:
        out = torch.empty_like(a)
    _call("pfd_add_rowvec_f16", a, row, a.numel() // C, C, out)
    return out


def ddim_step(eps: torch.Tensor, x: torch.Tensor, guidance: float, coef: torch.Tensor,
              step: Optional[torch.Tensor], x_prev: torch.Tensor, pred_x0: Optional[torch.Tensor], *,
              noise: Optional[torch.Tensor] = None, temperature: float = 1.0,
              log_tab: Optional[torch.Tensor] = None, log_xt: Optional[torch.Tensor] = None,
              log_x0: Optional[torch.Tensor] = None) -> None:
    """Fused CFG combine + DDIM update (see pfd_ddim_step_f16); eps holds [uncond | cond] halves."""
    _call("pfd_ddim_step_f16", eps, x, x.numel(), guidance, coef, step, x_prev, pred_x0, noise, float(temperature),
          log_tab, log_xt, log_x0)


def ddim_begin_step(step: torch.Tensor, ttab: torch.Tensor, t_out: torch.Tensor) -> None:
    """Device-side loop header: step -= 1; t_out[:] = ttab[step] (see pfd_ddim_begin_step)."""
    if step.dtype != torch.int32 or ttab.dtype != torch.int64 or t_out.dtype != torch.int64:
        raise RuntimeError("ddim_begin_step: step int32, ttab / t_out int64 expected")
    _call("pfd_ddim_begin_step", step, ttab, t_out, t_out.numel())


def ksampler_step(eps: torch.Tensor, cfg: bool, guidance: float, coef: torch.Tensor, step: torch.Tensor,
                  last_step: int, x: torch.Tensor, d_prev: torch.Tensor, unet_in: torch.Tensor, out: torch.Tensor, *,
                  noise: Optional[torch.Tensor] = None, log_tab: Optional[torch.Tensor] = None,
                  log_xt: Optional[torch.Tensor] = None, log_x0: Optional[torch.Tensor] = None) -> None:
    """One k-sampler step (see pfd_ksampler_step_f32): CFG combine, D = x - sigma*e, x = a*x + b*D + c*d_prev + u*noise,
    d_prev = D, unet_in = fp16(x*c_in_next) (both CFG halves), out = fp16(x) on the last step."""
    half_n = x.numel()
    _chk16(eps, "ksampler_step eps")
    for t, name in ((x, "x"), (d_prev, "d_prev"), (coef, "coef")):
        _chk32(t, f"ksampler_step {name}")
    if step.dtype != torch.int32 or coef.dim() != 2 or coef.shape[1] != PFD_KSAMPLER_NCOEF:
        raise RuntimeError("ksampler_step: int32 step and a [steps, 6] coefficient table expected")
    halves = 2 if cfg else 1
    if eps.numel() != halves * half_n or unet_in.numel() != halves * half_n or out.numel() != half_n \
            or d_prev.numel() != half_n or (noise is not None and noise.numel() != half_n):
        raise RuntimeError("ksampler_step: eps / unet_in / out / d_prev / noise sizes do not match the state")
    _chk16(unet_in, "ksampler_step unet_in")
    _chk16(out, "ksampler_step out")
    if noise is not None:
        _chk16(noise, "ksampler_step noise")
    _call("pfd_ksampler_step_f32", eps, int(cfg), float(guidance), half_n, coef, step, int(last_step), x, d_prev, noise,
          unet_in, out, log_tab, log_xt, log_x0)


def ksampler_begin_step(step: torch.Tensor, ttab: torch.Tensor, t_out: torch.Tensor) -> None:
    """Device-side loop header: step += 1; t_out[:] = ttab[step] (see pfd_ksampler_begin_step)."""
    if step.dtype != torch.int32 or ttab.dtype != torch.float32 or t_out.dtype != torch.float32:
        raise RuntimeError("ksampler_begin_step: step int32, ttab / t_out float32 expected")
    _call("pfd_ksampler_begin_step", step, ttab, ttab.numel(), t_out, t_out.numel())


def randn_f16(out: torch.Tensor, seeds: torch.Tensor, stream_id: int, draw: int = 0,
              draw_dev: Optional[torch.Tensor] = None, scale: float = 1.0) -> torch.Tensor:
    """out [B, ...] fp16 = scale * counter-based N(0, 1) noise of sample b from seeds[b] (see pfd_randn_f16).
    seeds: CUDA int64 [B] holding the uint64 seeds' bits; draw_dev (optional): CUDA int32 [1] added to draw."""
    _chk16(out, "randn_f16 out")
    if not out.is_contiguous() or out.dim() < 1:
        raise RuntimeError("randn_f16: out must be a contiguous [B, ...] tensor")
    B = out.shape[0]
    if seeds.dtype != torch.int64 or not seeds.is_cuda or not seeds.is_contiguous() or seeds.numel() != B:
        raise RuntimeError(f"randn_f16: seeds must be a contiguous CUDA int64 tensor of {B} entries")
    if draw_dev is not None and (draw_dev.dtype != torch.int32 or not draw_dev.is_cuda):
        raise RuntimeError("randn_f16: draw_dev must be a CUDA int32 tensor")
    _call("pfd_randn_f16", out, B, out.numel() // B, seeds, int(stream_id) & 0xffffffff, int(draw), draw_dev,
          float(scale))
    return out


def vae_posterior(moments: torch.Tensor, zc: int, *, noise: Optional[torch.Tensor] = None, scale: float = 1.0,
                  want=("mean", "logvar", "std", "sample")):
    """moments: channel-last [B,H,W,cpad] fp16 -> dict of NCHW fp16 [B,zc,H,W] tensors (pfd_vae_posterior_f16)."""
    B, H, W, cpad = moments.shape
    outs = {k: torch.empty((B, zc, H, W), device=moments.device, dtype=torch.float16) for k in want}
    if noise is not None and (noise.dtype != torch.float32 or not noise.is_contiguous()):
        noise = noise.to(torch.float32).contiguous()
    _call("pfd_vae_posterior_f16", moments, B, zc, H, W, cpad, noise, scale, outs.get("mean"), outs.get("logvar"),
          outs.get("std"), outs.get("sample"))
    return outs


def canny(x: torch.Tensor, low: int = 100, high: int = 200) -> Tuple[torch.Tensor, int]:
    """NCHW [B,3,H,W] image in [0,1] (fp16/fp32) -> (float32 [B,3,H,W] edge map, hysteresis sweeps).  Bit-exact
    cv2.Canny(ToPILImage(x), low, high) (pfd_canny_f32); synchronises the stream."""
    x, f32 = _chk_image(x, "canny")
    B, _, H, W = x.shape
    ws = torch.empty(int(load().pfd_canny_workspace_bytes(B, H, W)), device=x.device, dtype=torch.uint8)
    out = torch.empty((B, 3, H, W), device=x.device, dtype=torch.float32)
    sweeps = c_int32(0)
    _call("pfd_canny_f32", x, f32, B, H, W, int(low), int(high), ws, out, ctypes.byref(sweeps))
    return out, int(sweeps.value)


def image_u8_roundtrip(x: torch.Tensor) -> torch.Tensor:
    """ToTensor(ToPILImage(x)) = floor(x*255)/255 as float32 (pfd_image_u8_roundtrip_f32)."""
    if not x.is_cuda or x.dtype not in (torch.float16, torch.float32):
        raise RuntimeError("image_u8_roundtrip: expected a CUDA fp16/fp32 tensor")
    x = x.contiguous()
    out = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    _call("pfd_image_u8_roundtrip_f32", x, int(x.dtype == torch.float32), x.numel(), out)
    return out


def hed_input(x: torch.Tensor, norm: torch.Tensor, scale: float, cpad: int = 3) -> torch.Tensor:
    """NCHW [B,3,H,W] image in [0,1] (fp16/fp32) -> channel-last fp16 [B,H,W,cpad] = (x.mul(255).byte() - norm) * scale,
    zero pad channels (pfd_hed_input_f16).  norm: CUDA fp32 [3]."""
    x, f32 = _chk_image(x, "hed_input")
    _chk32(norm, "hed_input norm")
    B, _, H, W = x.shape
    out = torch.empty((B, H, W, cpad), device=x.device, dtype=torch.float16)
    _call("pfd_hed_input_f16", x, f32, B, H, W, cpad, norm, float(scale), out)
    return out


def hed_pool_side(x: torch.Tensor, proj_w: torch.Tensor, proj_b: torch.Tensor, pool: bool = True):
    """Block output x [B,h,w,C] fp16 -> (side [B,h,w] fp32 = x . proj_w + proj_b, 2x2 max-pooled [B,h/2,w/2,C] fp16 or
    None), both from one read of x (pfd_hed_pool_side_f16).  proj_w: CUDA fp32 [C]; proj_b: CUDA fp32 [1]."""
    _chk16(x, "hed_pool_side x")
    _chk32(proj_w, "hed_pool_side proj_w")
    _chk32(proj_b, "hed_pool_side proj_b")
    x = x.contiguous()
    B, h, w, C = x.shape
    if proj_w.numel() != C:
        raise RuntimeError(f"hed_pool_side: proj_w has {proj_w.numel()} entries for C={C}")
    side = torch.empty((B, h, w), device=x.device, dtype=torch.float32)
    pooled = torch.empty((B, h // 2, w // 2, C), device=x.device, dtype=torch.float16) if pool else None
    _call("pfd_hed_pool_side_f16", x, B, h, w, C, proj_w, proj_b, side, pooled)
    return side, pooled


def hed_fuse(sides: Sequence[torch.Tensor], H: int, W: int, inv_scale: float = 1.0) -> torch.Tensor:
    """apply_hed after the network: fp32 side maps [B,h_k,w_k] -> float32 [B,3,H,W] (pfd_hed_fuse_f32)."""
    n = len(sides)
    if not 1 <= n <= PFD_HED_MAX_SIDES:
        raise RuntimeError(f"hed_fuse: {n} side maps (1..{PFD_HED_MAX_SIDES})")
    B = sides[0].shape[0]
    for s in sides:
        _chk32(s, "hed_fuse side map")
        if s.dim() != 3 or s.shape[0] != B:
            raise RuntimeError(f"hed_fuse: side maps must be [B,h,w] with B={B}, got {tuple(s.shape)}")
    out = torch.empty((B, 3, H, W), device=sides[0].device, dtype=torch.float32)
    ptrs = (c_void_p * n)(*[s.data_ptr() for s in sides])
    hs = (c_int32 * n)(*[s.shape[1] for s in sides])
    ws = (c_int32 * n)(*[s.shape[2] for s in sides])
    _call("pfd_hed_fuse_f32", ptrs, hs, ws, n, B, H, W, float(inv_scale), out)
    return out


def scribble_hed(hed: torch.Tensor, return_nms: bool = False):
    """make_scribble of the HED map: float32 [B,3,H,W] (pfd_hed_fuse_f32's output; channel 0 is read as the levels
    round(255 * v)) -> float32 [B,3,H,W] scribble map (pfd_scribble_hed_f32).  return_nms=True also returns the uint8
    [B,H,W] map after the non-maximum suppression and the `> 127` threshold."""
    _chk32(hed, "scribble_hed")
    if hed.dim() != 4 or hed.shape[1] < 1:
        raise RuntimeError(f"scribble_hed: expected [B,C,H,W], got {tuple(hed.shape)}")
    B, C, H, W = hed.shape
    nms = torch.empty((B, H, W), device=hed.device, dtype=torch.uint8)
    out = torch.empty((B, 3, H, W), device=hed.device, dtype=torch.float32)
    _call("pfd_scribble_hed_f32", hed, C * H * W, B, H, W, nms, out)
    return (out, nms) if return_nms else out


def scribble_blur_u8(z: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """cv2.GaussianBlur(z, (0,0), 3) of a CUDA uint8 [B,H,W] map, bit-exact -> (blurred uint8 [B,H,W], float32
    [B,3,H,W] with 1.0 where blurred > 4) (pfd_scribble_blur_u8)."""
    if z.dim() != 3 or z.dtype != torch.uint8 or not z.is_cuda:
        raise RuntimeError(f"scribble_blur_u8: expected a CUDA uint8 [B,H,W] map, got {tuple(z.shape)} {z.dtype}")
    z = z.contiguous()
    B, H, W = z.shape
    blurred = torch.empty_like(z)
    out = torch.empty((B, 3, H, W), device=z.device, dtype=torch.float32)
    _call("pfd_scribble_blur_u8", z, B, H, W, blurred, out)
    return blurred, out


def scribble_xdog(x: torch.Tensor, threshold: int = 32) -> torch.Tensor:
    """The xdog scribble of an NCHW [B,3,H,W] image in [0,1] (fp16/fp32) -> float32 [B,3,H,W]
    (pfd_scribble_xdog_f32).  threshold: integer; the uint8 edge strength is compared with `>`."""
    x, f32 = _chk_image(x, "scribble_xdog")
    B, _, H, W = x.shape
    out = torch.empty((B, 3, H, W), device=x.device, dtype=torch.float32)
    _call("pfd_scribble_xdog_f32", x, f32, B, H, W, int(threshold), out)
    return out


def pidinet_dw(x: torch.Tensor, w: torch.Tensor, pool: bool = False):
    """Depthwise conv1 of a PiDiNet block: channel-last x [B,H,W,C] fp16, w CUDA fp32 [ks*ks, C] (ks 3 or 5) ->
    relu(conv) [B,h,w,C] fp16, and with pool=True (ks 3) the 2x2 max-pooled input it convolved, [B,H/2,W/2,C]
    (pfd_pidinet_dw_f16)."""
    _chk16(x, "pidinet_dw x")
    _chk32(w, "pidinet_dw w")
    x = x.contiguous()
    B, H, W, C = x.shape
    ks = {9: 3, 25: 5}.get(w.shape[0], 0)
    if w.dim() != 2 or w.shape[1] != C or not ks:
        raise RuntimeError(f"pidinet_dw: weights {tuple(w.shape)} do not fit C={C}")
    h, wd = (H // 2, W // 2) if pool else (H, W)
    out = torch.empty((B, h, wd, C), device=x.device, dtype=torch.float16)
    pooled = torch.empty_like(out) if pool else None
    _call("pfd_pidinet_dw_f16", x, B, H, W, C, ks, int(pool), w, out, pooled)
    return (out, pooled) if pool else out


def pidinet_reduce(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """CDCM's relu + 1x1 conv to 24 channels: x [B,h,w,C] fp16, w CUDA fp32 [C, 24], b [24] -> [B,h,w,24] fp16
    (pfd_pidinet_reduce_f16)."""
    _chk16(x, "pidinet_reduce x")
    _chk32(w, "pidinet_reduce w")
    _chk32(b, "pidinet_reduce b")
    x = x.contiguous()
    B, h, wd, C = x.shape
    if tuple(w.shape) != (C, 24) or b.numel() != 24:
        raise RuntimeError(f"pidinet_reduce: weights {tuple(w.shape)} / bias {tuple(b.shape)} do not fit C={C}")
    m = torch.empty((B, h, wd, 24), device=x.device, dtype=torch.float16)
    _call("pfd_pidinet_reduce_f16", x, B * h * wd, C, w, b, m)
    return m


def pidinet_cdcm(m: torch.Tensor, wpk: torch.Tensor) -> torch.Tensor:
    """Sum of CDCM's four dilated 3x3 convs: m [B,h,w,24] fp16, wpk the packed fragments (pidinet.pack_cdcm) ->
    [B,h,w,24] fp32 (pfd_pidinet_cdcm_f16)."""
    _chk16(m, "pidinet_cdcm m")
    _chk16(wpk, "pidinet_cdcm wpk")
    m = m.contiguous()
    B, h, w, C = m.shape
    if C != 24 or wpk.numel() != 54 * 3 * 32 * 4:
        raise RuntimeError(f"pidinet_cdcm: m {tuple(m.shape)} / packed weights {wpk.numel()} do not fit")
    u = torch.empty((B, h, w, 24), device=m.device, dtype=torch.float32)
    _call("pfd_pidinet_cdcm_f16", m, B, h, w, wpk, u)
    return u


def pidinet_side(u: torch.Tensor, params: torch.Tensor) -> torch.Tensor:
    """CSAM + MapReduce of a stage: u [B,h,w,24] fp32 -> side map [B,h,w] fp32 (pfd_pidinet_side_f32)."""
    _chk32(u, "pidinet_side u")
    _chk32(params, "pidinet_side params")
    B, h, w, C = u.shape
    if C != 24 or params.numel() != PFD_PIDINET_SIDE_PARAMS:
        raise RuntimeError(f"pidinet_side: u {tuple(u.shape)} / params {params.numel()} do not fit")
    side = torch.empty((B, h, w), device=u.device, dtype=torch.float32)
    _call("pfd_pidinet_side_f32", u, B, h, w, params, side)
    return side


def pidinet_fuse(sides: Sequence[torch.Tensor], cls: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Four fp32 side maps [B,h_k,w_k] -> float32 [B,3,H,W] levels / 255 (pfd_pidinet_fuse_f32).  cls: CUDA fp32 [5]
    = classifier weights, bias."""
    if len(sides) != 4:
        raise RuntimeError(f"pidinet_fuse: {len(sides)} side maps (4 expected)")
    _chk32(cls, "pidinet_fuse cls")
    B = sides[0].shape[0]
    for s in sides:
        _chk32(s, "pidinet_fuse side map")
        if s.dim() != 3 or s.shape[0] != B:
            raise RuntimeError(f"pidinet_fuse: side maps must be [B,h,w] with B={B}, got {tuple(s.shape)}")
    out = torch.empty((B, 3, H, W), device=sides[0].device, dtype=torch.float32)
    ptrs = (c_void_p * 4)(*[s.data_ptr() for s in sides])
    hs = (c_int32 * 4)(*[s.shape[1] for s in sides])
    ws = (c_int32 * 4)(*[s.shape[2] for s in sides])
    _call("pfd_pidinet_fuse_f32", ptrs, hs, ws, B, H, W, cls, out)
    return out


def mlsd_input(x: torch.Tensor) -> torch.Tensor:
    """NCHW [B,3,H,W] image in [0,1] (fp16/fp32) -> channel-last fp16 [B,H,W,16] = [u8 - 127.5 (rgb), 1 - 127.5, 0 x 12]
    with u8 = x.mul(255).byte() (pfd_mlsd_input_f16)."""
    x, f32 = _chk_image(x, "mlsd_input")
    B, _, H, W = x.shape
    out = torch.empty((B, H, W, 16), device=x.device, dtype=torch.float16)
    _call("pfd_mlsd_input_f16", x, f32, B, H, W, out)
    return out


def mlsd_dw(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, stride: int) -> torch.Tensor:
    """Depthwise 3x3 ConvBNReLU6 of channel-last x [B,H,W,C] fp16 (min(x, 6) on the input), w CUDA fp32 [9, C], b [C];
    stride 2 pads like TFLite -> [B,H/s,W/s,C] fp16 (pfd_mlsd_dw_f16)."""
    _chk16(x, "mlsd_dw x")
    _chk32(w, "mlsd_dw w")
    _chk32(b, "mlsd_dw b")
    x = x.contiguous()
    B, H, W, C = x.shape
    if tuple(w.shape) != (9, C) or b.numel() != C:
        raise RuntimeError(f"mlsd_dw: weights {tuple(w.shape)} / bias {tuple(b.shape)} do not fit C={C}")
    out = torch.empty((B, H // stride, W // stride, C), device=x.device, dtype=torch.float16)
    _call("pfd_mlsd_dw_f16", x, B, H, W, C, int(stride), w, b, out)
    return out


def mlsd_upsample(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Bilinear x2 (align_corners=True) of x [B,h,w,C] fp16 into out, a [B,2h,2w,C] view whose pixels are out.stride(2)
    elements apart (e.g. a channel slice of a concat buffer) (pfd_mlsd_upsample_f16)."""
    _chk16(x, "mlsd_upsample x")
    _chk16(out, "mlsd_upsample out")
    x = x.contiguous()
    B, h, w, C = x.shape
    p = out.stride(2)
    if tuple(out.shape) != (B, 2 * h, 2 * w, C) or out.stride(3) != 1 or out.stride(1) != 2 * w * p \
            or out.stride(0) != 2 * h * out.stride(1):
        raise RuntimeError(f"mlsd_upsample: out {tuple(out.shape)} / strides {out.stride()} do not fit x {tuple(x.shape)}")
    _call("pfd_mlsd_upsample_f16", x, B, h, w, C, out, p)
    return out


def mlsd_head(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """x [B,h,w,C] fp16 -> fp32 [B,5,h,w] = w . x + b, w CUDA fp32 [5, C], b [5] (pfd_mlsd_head_f32)."""
    _chk16(x, "mlsd_head x")
    _chk32(w, "mlsd_head w")
    _chk32(b, "mlsd_head b")
    x = x.contiguous()
    B, h, wd, C = x.shape
    if tuple(w.shape) != (5, C) or b.numel() != 5:
        raise RuntimeError(f"mlsd_head: weights {tuple(w.shape)} / bias {tuple(b.shape)} do not fit C={C}")
    out = torch.empty((B, 5, h, wd), device=x.device, dtype=torch.float32)
    _call("pfd_mlsd_head_f32", x, B, h, wd, C, w, b, out)
    return out


def mlsd_decode(maps: torch.Tensor, thr_v: float, thr_d: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 maps [B,5,h,w] (centre logit, start / end displacements) -> (int32 segments [B,200,4] (x0, y0, x1, y1),
    int32 counts [B]) on the device (pfd_mlsd_decode_f32); rows past count[n] are unspecified."""
    _chk32(maps, "mlsd_decode maps")
    if maps.dim() != 4 or maps.shape[1] != 5:
        raise RuntimeError(f"mlsd_decode: expected [B,5,h,w] maps, got {tuple(maps.shape)}")
    B, _, h, w = maps.shape
    keys = torch.empty((B, h, w), device=maps.device, dtype=torch.int32)
    segs = torch.empty((B, PFD_MLSD_TOPK, 4), device=maps.device, dtype=torch.int32)
    count = torch.empty((B,), device=maps.device, dtype=torch.int32)
    _call("pfd_mlsd_decode_f32", maps, B, h, w, float(thr_v), float(thr_d), keys, segs, count)
    return segs, count


def mlsd_draw(segs: torch.Tensor, count: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """float32 [B,3,H,W], 1.0 on the cv2.line(..., 1, LINE_8) pixels of segs[n, :count[n]] (int32 [B,200,4], device
    counts) and 0 elsewhere (pfd_mlsd_draw_f32)."""
    if segs.dtype != torch.int32 or count.dtype != torch.int32 or not segs.is_cuda or not count.is_cuda \
            or segs.dim() != 3 or tuple(segs.shape[1:]) != (PFD_MLSD_TOPK, 4) or count.numel() != segs.shape[0]:
        raise RuntimeError(f"mlsd_draw: expected CUDA int32 segments [B,{PFD_MLSD_TOPK},4] and counts [B]")
    segs, count = segs.contiguous(), count.contiguous()
    B = segs.shape[0]
    out = torch.zeros((B, 3, H, W), device=segs.device, dtype=torch.float32)
    _call("pfd_mlsd_draw_f32", segs, count, B, H, W, out)
    return out


def openpose_input(x: torch.Tensor, h: int, w: int, hp: int, wp: int, plan, tabs) -> torch.Tensor:
    """NCHW [B,3,H,W] image in [0,1] -> channel-last fp16 [B,hp,wp,16]: u8 = x.mul(255).byte(), BGR, cv2.resize to
    h x w by ``plan`` (openpose_tables.resize_plan; ``tabs`` its device tables), 128 pad, u8 / 256 - 0.5
    (pfd_openpose_input_f16)."""
    x, f32 = _chk_image(x, "openpose_input")
    B, _, H, W = x.shape
    out = torch.empty((B, hp, wp, 16), device=x.device, dtype=torch.float16)
    mode, fy, fx, ay, ax = _plan_args(plan, tabs, u8=True)
    _call("pfd_openpose_input_f16", x, f32, B, H, W, h, w, hp, wp, mode, fy, fx, *ay, *ax, out)
    return out


def _plan_args(plan, tabs, u8: bool = False):
    """(mode, fy, fx, (iy, wy, ty), (ix, wx, tx)) of a resize plan for the openpose kernels."""
    none = (None, None, 0)
    if plan[0] == "copy":
        return 0, 0, 0, none, none
    if plan[0] == "block":
        return 1, plan[1], plan[2], none, none
    (iy, wy), (ix, wx) = tabs
    mode = (2 if wy.dtype == torch.int32 else 3) if u8 else 2
    return mode, 0, 0, (iy, wy, iy.shape[1]), (ix, wx, ix.shape[1])


def openpose_pool(x: torch.Tensor) -> torch.Tensor:
    """2x2 / stride 2 max pool of x [B,H,W,C] fp16 (pfd_openpose_pool_f16)."""
    _chk16(x, "openpose_pool x")
    x = x.contiguous()
    B, H, W, C = x.shape
    out = torch.empty((B, H // 2, W // 2, C), device=x.device, dtype=torch.float16)
    _call("pfd_openpose_pool_f16", x, B, H, W, C, out)
    return out


def im2col7x7(x: torch.Tensor) -> torch.Tensor:
    """x [B,H,W,C] fp16 -> [B*H*W, 49*C] rows of the 7x7 / pad 3 neighbourhood, k = tap * C + c (pfd_im2col7x7_f16)."""
    _chk16(x, "im2col7x7 x")
    x = x.contiguous()
    B, H, W, C = x.shape
    out = torch.empty((B * H * W, 49 * C), device=x.device, dtype=torch.float16)
    _call("pfd_im2col7x7_f16", x, B, H, W, C, out)
    return out


def openpose_head(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, relu: bool, out: torch.Tensor, off: int) -> None:
    """out[:, off:off+N] (planar fp32 [B,C_out,h,w]) = act(w . x + b) of x [B,h,w,C] fp16, w fp32 [N, C]
    (pfd_openpose_head_f32)."""
    _chk16(x, "openpose_head x")
    _chk32(w, "openpose_head w")
    _chk32(b, "openpose_head b")
    _chk32(out, "openpose_head out")
    x = x.contiguous()
    B, h, wd, C = x.shape
    N = w.shape[0]
    if w.shape[1] != C or b.numel() != N or out.shape[0] != B or tuple(out.shape[2:]) != (h, wd):
        raise RuntimeError(f"openpose_head: weights {tuple(w.shape)} / out {tuple(out.shape)} do not fit x {tuple(x.shape)}")
    _call("pfd_openpose_head_f32", x, B, h, wd, C, w, b, N, int(relu), out, out.shape[1], off)


def openpose_resize(src: torch.Tensor, c0: int, C: int, H: int, W: int, plan, tabs) -> torch.Tensor:
    """cv2.resize of channels c0..c0+C of planar fp32 src [B,Cs,hs,ws] to [B,C,H,W] (pfd_openpose_resize_f32); a
    'copy' plan to a smaller H x W is the top-left crop."""
    _chk32(src, "openpose_resize src")
    B, Cs, hs, ws = src.shape
    out = torch.empty((B, C, H, W), device=src.device, dtype=torch.float32)
    mode, fy, fx, ay, ax = _plan_args(plan, tabs)
    _call("pfd_openpose_resize_f32", src, B, Cs, c0, C, hs, ws, H, W, mode, fy, fx, *ay, *ax, out)
    return out


def openpose_peaks(maps: torch.Tensor, gauss: torch.Tensor):
    """Heatmaps fp32 [B,18,H,W] -> (xy int32 [B,18,MAX_PEAKS,2], score float64 [B,18,MAX_PEAKS], total int32 [B,18])
    after the float64 Gaussian (gauss: CUDA float64 [13]) (pfd_openpose_peaks_f32)."""
    _chk32(maps, "openpose_peaks maps")
    B, P, H, W = maps.shape
    if P != 18 or gauss.dtype != torch.float64 or gauss.numel() != 13:
        raise RuntimeError(f"openpose_peaks: expected [B,18,H,W] maps and 13 float64 weights, got {tuple(maps.shape)}")
    dev = maps.device
    tmp = torch.empty((B, 18, H, W), device=dev, dtype=torch.float64)
    blur = torch.empty_like(tmp)
    rowcnt = torch.empty((B * 18 * H,), device=dev, dtype=torch.int32)
    xy = torch.zeros((B, 18, PFD_OPENPOSE_MAX_PEAKS, 2), device=dev, dtype=torch.int32)
    score = torch.zeros((B, 18, PFD_OPENPOSE_MAX_PEAKS), device=dev, dtype=torch.float64)
    total = torch.empty((B, 18), device=dev, dtype=torch.int32)
    _call("pfd_openpose_peaks_f32", maps, B, H, W, gauss, tmp, blur, rowcnt, xy, score, total)
    return xy, score, total


def openpose_assemble(up: torch.Tensor, H: int, W: int, plan, tabs, total: torch.Tensor, xy: torch.Tensor,
                      score: torch.Tensor):
    """PAF scoring, limb matching and person assembly (pfd_openpose_assemble_f32) -> (persons int32 [B,MAX_PERSONS,18],
    pscore float64 [B,MAX_PERSONS,2], npersons int32 [B]).  up: planar fp32 [B,57,hs,ws]."""
    _chk32(up, "openpose_assemble up")
    B, C, hs, ws = up.shape
    dev = up.device
    P, R = PFD_OPENPOSE_MAX_PEAKS, PFD_OPENPOSE_MAX_PERSONS
    conn = torch.empty((B, 19, P * P), device=dev, dtype=torch.float64)
    rows = torch.empty((B, R, 20), device=dev, dtype=torch.float64)
    persons = torch.empty((B, R, 18), device=dev, dtype=torch.int32)
    pscore = torch.empty((B, R, 2), device=dev, dtype=torch.float64)
    npersons = torch.empty((B,), device=dev, dtype=torch.int32)
    mode, fy, fx, ay, ax = _plan_args(plan, tabs)
    _call("pfd_openpose_assemble_f32", up, B, C, hs, ws, H, W, mode, fy, fx, *ay, *ax, total, xy, score, conn, rows,
          persons, pscore, npersons)
    return persons, pscore, npersons


def openpose_draw(persons: torch.Tensor, npersons: torch.Tensor, xy: torch.Tensor, H: int, W: int,
                  sintab: torch.Tensor, colors: torch.Tensor) -> torch.Tensor:
    """util.draw_bodypose of every person -> float32 [B,3,H,W] canvas / 255 (pfd_openpose_draw_f32)."""
    B = persons.shape[0]
    dev = persons.device
    idx = torch.empty((B, H, W), device=dev, dtype=torch.int32)
    out = torch.empty((B, 3, H, W), device=dev, dtype=torch.float32)
    _call("pfd_openpose_draw_f32", persons, npersons, xy, B, H, W, sintab, colors, idx, out)
    return out


def window_gather(x: torch.Tensor, ws: int, shift: int) -> torch.Tensor:
    B, H, W, C = x.shape
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    out = torch.empty((B * (Hp // ws) * (Wp // ws), ws * ws, C), device=x.device, dtype=torch.float16)
    _call("pfd_window_gather_f16", x, B, H, W, C, ws, shift, out)
    return out


def window_scatter(win: torch.Tensor, B: int, H: int, W: int, ws: int, shift: int,
                   residual: Optional[torch.Tensor]) -> torch.Tensor:
    C = win.shape[-1]
    out = torch.empty((B, H, W, C), device=win.device, dtype=torch.float16)
    _call("pfd_window_scatter_f16", win, B, H, W, C, ws, shift, residual, out)
    return out


def patch_merge_gather(x: torch.Tensor) -> torch.Tensor:
    B, H, W, C = x.shape
    out = torch.empty((B, (H + 1) // 2, (W + 1) // 2, 4 * C), device=x.device, dtype=torch.float16)
    _call("pfd_patch_merge_gather_f16", x, B, H, W, C, out)
    return out


def patchify(img: torch.Tensor, P: int, kpad: int) -> torch.Tensor:
    """NCHW image (fp16/fp32) -> [B, ceil(H/P), ceil(W/P), kpad] patch rows (see pfd_patchify_f16)."""
    B, C, H, W = img.shape
    img = img.contiguous()
    if img.dtype not in (torch.float16, torch.float32):
        img = img.to(torch.float16)
    out = torch.empty((B, -(-H // P), -(-W // P), kpad), device=img.device, dtype=torch.float16)
    _call("pfd_patchify_f16", img, int(img.dtype == torch.float32), B, C, H, W, P, kpad, out)
    return out


def _check_flash_shapes(what: str, q_rows: int, k_rows: int, k_d: int, vt_d: int, vt_cols: int, d: int, Nq: int,
                        Nk: int) -> None:
    # the kernel's tensor maps take Nq / Nk rows and d channels per head at the given strides: anything beyond a
    # head's rows is the next head's data (or past the allocation for the last head)
    if not (0 < Nq <= q_rows and 0 < Nk <= min(k_rows, vt_cols)):
        raise ValueError(f"{what}: Nq={Nq}, Nk={Nk} exceed q rows {q_rows}, k rows {k_rows} or V^T columns {vt_cols}")
    if k_d != d or vt_d != d:
        raise ValueError(f"{what}: head dims differ: q {d}, k {k_d}, V^T rows {vt_d}")


def _check_flash_out(what: str, out: torch.Tensor, B: int, heads: int, Nq: int, d: int) -> None:
    # the epilogue stores __half2 pairs at out + b*stride(0) + q*stride(1) + h*d + c (c even)
    _chk16(out, f"{what}: out")
    if (out.dim() != 3 or out.shape[0] != B or out.shape[1] < Nq or out.shape[2] < heads * d
            or out.stride(2) != 1 or out.stride(0) % 2 or out.stride(1) % 2 or out.data_ptr() % 4):
        raise ValueError(f"{what}: out must be a [{B}, >={Nq}, >={heads * d}] view with unit column stride, even row "
                         f"and batch strides and a 4-byte aligned base, got {tuple(out.shape)} with strides "
                         f"{out.stride()} at offset {out.storage_offset()}")


def flash_attn(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, *, B: int, heads: int, Nq: int, Nk: int,
               scale: float, out: torch.Tensor) -> torch.Tensor:
    """Fused attention (see pfd_flash_attn_f16): q [BH, Nqp, d], k [BH, Nkp, d], vt [BH, d, Nkp] ->
    out [B, Nq, heads*d]."""
    for t, name in ((q, "q"), (k, "k"), (vt, "vt")):
        _chk16(t, f"flash_attn: {name}")
        if t.dim() != 3 or t.shape[0] != B * heads or not t.is_contiguous():
            raise ValueError(f"flash_attn: {name} must be a contiguous [B*heads={B * heads}, rows, cols] tensor, "
                             f"got {tuple(t.shape)} with strides {t.stride()}")
    d = q.shape[2]
    _check_flash_shapes("flash_attn", q.shape[1], k.shape[1], k.shape[2], vt.shape[1], vt.shape[2], d, Nq, Nk)
    _check_flash_out("flash_attn", out, B, heads, Nq, d)
    _call("pfd_flash_attn_f16", q, k, vt, out, B, heads, Nq, Nk, d, q.shape[1], k.shape[1], scale, vt.shape[2],
          out.stride(0), out.stride(1), 0)
    return out


def flash_attn_strided(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, *, Nq: int, Nk: int, scale: float,
                       out: torch.Tensor) -> torch.Tensor:
    """pfd_flash_attn_strided_f16: q, k strided views [B, heads, N(p), d]; vt strided view [B, heads, d, Nk(p)]
    (rows contiguous); out [B, Nq, heads*d]."""
    for t, name in ((q, "q"), (k, "k"), (vt, "vt")):
        _chk16(t, f"flash_attn_strided: {name}")
        if t.dim() != 4 or t.shape[:2] != q.shape[:2] or t.stride(3) != 1:
            raise ValueError(f"flash_attn_strided: {name} must be a [{', '.join(map(str, q.shape[:2]))}, rows, cols] "
                             f"view with unit column stride, got {tuple(t.shape)} with strides {t.stride()}")
    B, heads, _, d = q.shape
    _check_flash_shapes("flash_attn_strided", q.shape[2], k.shape[2], k.shape[3], vt.shape[2], vt.shape[3], d, Nq, Nk)
    _check_flash_out("flash_attn_strided", out, B, heads, Nq, d)
    st = lambda t: (c_int64 * 3)(t.stride(0), t.stride(1), t.stride(2))
    _call("pfd_flash_attn_strided_f16", q, k, vt, out, B, heads, Nq, Nk, d, st(q), st(k), st(vt), scale, out.stride(0),
          out.stride(1))
    return out
