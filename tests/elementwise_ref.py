"""References, error bounds and kernel models for the elementwise tests (test_elementwise_gpu.py and its CPU model
test_elementwise_model_cpu.py).  This module holds no tests.

DDIM update (pfd_b200/csrc/elementwise.cu, ddim_step_kernel).  ``ddim_eager`` is the reference step (ddim.py:150-170)
written as torch fp16 operations on whatever device its inputs live on, so it rounds exactly as the reference does:
every tensor op is computed in fp32 and rounded to fp16, and python scalars (guidance, temperature) stay fp32.  The
kernel must reproduce it bit for bit.  ``ddim_kernel_model`` is a numpy float32 emulation of the kernel's arithmetic
with switches for subtly wrong variants.

GELU epilogue (pfd_b200/csrc/gemm_tc.cu, gelu_sig).  ``gelu_sig_model`` emulates x * sigmoid(x * poly(x^2)) in float32;
``gelu_sig_bound`` is its documented error against the exact erf GELU.

Swin window maps (window_gather_kernel / window_scatter_kernel).  ``window_gather_ref`` / ``window_scatter_ref`` are the
reference's pad -> roll -> partition and reverse -> roll -> crop (swin.py:269-304) as torch views;
``window_gather_index`` / ``window_scatter_index`` restate the kernels' index arithmetic in numpy.

Timestep embedding (timestep_embedding_kernel).  ``temb_ref`` is the float64 [cos | sin] embedding
(diffusion_utils.py:141-146) and its bound for the kernel's fp32 evaluation.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from attention_ref import ulp16

U32 = 2.0 ** -24             # fp32 unit roundoff
F32 = np.float32

DDIM_STEPS = 50
DDIM_GUIDANCE_CFG = (1.8, 2.0, 7.5)      # [uncond | cond] eps; 1.8 is not an fp16 value
DDIM_GUIDANCE_NOCFG = (1.0, 3.0)         # eps = [0 | e], the reference's e_t * scale (ddim.py:143-144)
DDIM_TEMPERATURES = (1.0, 0.5, 0.7, 0.9)
DDIM_MUTANTS = ("rh_temperature", "rh_guidance", "unrounded_diff", "dir_coef_unrounded")


# ------------------------------------------------------------------------------------------------- fp16 helpers
def half_rn(x: torch.Tensor) -> torch.Tensor:
    """float64 -> fp16 rounded once, to nearest even (a plain .half() goes through float32 and can round twice)."""
    q = ulp16(x)
    return (torch.round(x.double() / q) * q).to(torch.float16)


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


def bit_mismatch(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Elements whose fp16 bits differ, NaNs counting as equal to any NaN (their payload and sign are not part of the
    arithmetic: at eta = 1 the reference's fp16 1 - a_prev - sigma^2 is negative at schedule index 1, so its step is
    NaN there, and the kernel's must be too)."""
    a, b = a.reshape(-1), b.reshape(-1)
    return (bits(a) != bits(b)) & ~(torch.isnan(a) & torch.isnan(b))


def rh32(x):
    """numpy float32 -> fp16 -> float32 (the kernels' rh)."""
    return np.asarray(x, F32).astype(np.float16).astype(F32)


# ------------------------------------------------------------------------------------------------- DDIM
def ddim_schedule_sampler(eta: float, steps: int = DDIM_STEPS):
    """A DDIMSampler over the SD-v1.5 schedule buffers (pfd.py:110-160) with make_schedule(steps, eta) applied."""
    from oracle import pfd_oracle as O
    from pfd_b200.ddim import DDIMSampler
    buf = O.schedule_buffers()

    class Schedule:
        num_timesteps = 1000
        betas, alphas_cumprod, alphas_cumprod_prev = buf["betas"], buf["alphas_cumprod"], buf["alphas_cumprod_prev"]
        sqrt_one_minus_alphas_cumprod = buf["sqrt_one_minus_alphas_cumprod"]
    s = DDIMSampler(Schedule())
    s.make_schedule(steps, ddim_eta=eta, verbose=False)
    return s


def ddim_coefs(sampler, index: int, original: bool, device, ndim: int):
    """(a_t, a_prev, sigma_t, sqrt_one_minus_at) as the reference builds them (ddim.py:155-163): torch.full(...,
    dtype=float16) of the schedule entries at `index`, each taken from the attribute in the dtype make_schedule left
    it in (fp32 tensors, float64 numpy arrays)."""
    if original:
        m = sampler.model
        srcs = (m.alphas_cumprod, m.alphas_cumprod_prev, sampler.ddim_sigmas_for_original_num_steps,
                m.sqrt_one_minus_alphas_cumprod)
    else:
        srcs = (sampler.ddim_alphas, sampler.ddim_alphas_prev, sampler.ddim_sigmas, sampler.ddim_sqrt_one_minus_alphas)
    shape = [1] * ndim
    return tuple(torch.full(shape, s[index], device=device, dtype=torch.float16) for s in srcs)


def ddim_eager(eps, x, guidance, coefs, noise=None, temperature=1.0, cfg=True):
    """The reference step (ddim.py:140-170) in torch fp16.  eps: [uncond | cond] halves (cfg) or [0 | e] (not cfg:
    e_t = e * scale).  Returns (x_prev, pred_x0)."""
    a_t, a_prev, sigma_t, sqrt_one_minus_at = coefs
    e_u, e_c = eps.chunk(2)
    e_t = e_u + guidance * (e_c - e_u) if cfg else e_c * guidance
    pred_x0 = (x - sqrt_one_minus_at * e_t) / a_t.sqrt()
    dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
    x_prev = a_prev.sqrt() * pred_x0 + dir_xt
    if noise is not None:
        x_prev = x_prev + sigma_t * noise * temperature
    return x_prev, pred_x0


def ddim_kernel_model(eps, x, guidance, coef_row, noise=None, temperature=1.0, mutant=None):
    """numpy float32 emulation of ddim_step_kernel: eps [2n], x [n], noise [n] (fp16 values), coef_row the four fp32
    entries of one row of the coefficient table.  mutant: one of DDIM_MUTANTS, or None for the kernel as it is.
    Returns (x_prev, pred_x0) as fp16 arrays."""
    eps = np.asarray(eps, F32)
    n = eps.size // 2
    eu, ec = eps[:n], eps[n:]
    xv = np.asarray(x, F32)
    a_t, a_prev, sigma, s1m = (rh32(F32(c)) for c in coef_row)
    sqrt_at, sqrt_ap = rh32(np.sqrt(a_t)), rh32(np.sqrt(a_prev))
    with np.errstate(invalid="ignore"):                  # NaN where 1 - a_prev - sigma^2 < 0, as in the reference
        if mutant == "dir_coef_unrounded":
            dir_c = rh32(np.sqrt(F32(1) - a_prev - sigma * sigma))
        else:
            dir_c = rh32(np.sqrt(rh32(rh32(F32(1) - a_prev) - rh32(sigma * sigma))))
    g = rh32(F32(guidance)) if mutant == "rh_guidance" else F32(guidance)
    temp = rh32(F32(temperature)) if mutant == "rh_temperature" else F32(temperature)
    d = (ec - eu) if mutant == "unrounded_diff" else rh32(ec - eu)
    e = rh32(eu + rh32(g * d))
    p0 = rh32(rh32(xv - rh32(s1m * e)) / sqrt_at)
    xp = rh32(rh32(sqrt_ap * p0) + rh32(dir_c * e))
    if noise is not None:
        xp = rh32(xp + rh32(rh32(sigma * np.asarray(noise, F32)) * temp))
    return xp.astype(np.float16), p0.astype(np.float16)


def ddim_inputs(half_shape, scale, seed, cfg=True):
    """(eps [2, ...], x, noise) fp16 CPU tensors at `scale`; eps is [0 | e] without cfg.  All finite."""
    g = torch.Generator().manual_seed(seed)
    n = [2 * half_shape[0]] + list(half_shape[1:])
    eps = (torch.randn(n, generator=g) * scale).half()
    if not cfg:
        eps[:half_shape[0]] = 0
    x = (torch.randn(list(half_shape), generator=g) * scale).half()
    noise = torch.randn(list(half_shape), generator=g).half()
    return eps, x, noise


# ------------------------------------------------------------------------------------------------- timestep embedding
def temb_ref(t, dim: int, max_period: float):
    """t: float64 tensor [n] (the timesteps as the kernel sees them, i.e. fp32 values) -> (ref, bound), float64
    [n, dim]: the exact [cos | sin] (+ a zero column for odd dim) and the kernel's error bound.

    The kernel evaluates freq = expf(-logf(P) * i / half), arg = t * freq in fp32, then cosf / sinf and one fp16
    rounding.  With u = 2^-24: logf (1 ulp) is within 2u relative, the product and the quotient round once each (u
    each), so z = -ln(P) i / half carries a relative error of 4u; expf (2 ulp, 4u) then gives freq within (4 |z| + 4) u
    relative, and t * freq adds u: arg is within (4 |z| + 5) u |arg|.  cosf / sinf (2 ulp) add 4u of the result, and
    the fp16 rounding half an ulp of it (of the binade the fp32 value may have moved into).
    Bound = ulp16(|ref| + d) / 2 + d with d = (4 |z| + 5) u |arg| + 4u |ref|."""
    t = t.double()
    half = dim // 2
    i = torch.arange(half, dtype=torch.float64)
    z = -math.log(max_period) * i / half
    arg = t[:, None] * torch.exp(z)[None, :]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    d_arg = (4 * z.abs() + 5)[None, :] * U32 * arg.abs()
    d = torch.cat([d_arg, d_arg], 1) + 4 * U32 * ref.abs()
    bound = 0.5 * ulp16(ref.abs() + d) + d
    if dim % 2:
        ref = torch.cat([ref, torch.zeros_like(ref[:, :1])], 1)
        bound = torch.cat([bound, torch.zeros_like(bound[:, :1])], 1)
    return ref, bound


# ------------------------------------------------------------------------------------------------- GELU epilogue
GELU_SIG_COEF = (1.01426305e-3, -1.06775723e-1, -2.30112135)   # gemm_tc.cu gelu_sig, pre-multiplied by -log2(e)
GELU_FIT_ERR = 2.6e-5        # |gelu_sig - gelu| on [-10, 10]: the fit's 2.5e-5 plus the fp32 evaluation
GELU_CLAMP_REL = 3e-9        # beyond |x| = 10 the clamped sigmoid is off by at most 2.91e-9 (2^-28.36 at x = -10)


def gelu64(x: torch.Tensor) -> torch.Tensor:
    """Exact erf GELU in float64."""
    x = x.double()
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_sig_bound(g: torch.Tensor) -> torch.Tensor:
    """Bound of |gelu_sig(g) - gelu(g)| (float64)."""
    g = g.double().abs()
    return torch.where(g <= 10, torch.full_like(g, GELU_FIT_ERR), GELU_CLAMP_REL * g)


def gelu_sig_model(x, coef=GELU_SIG_COEF):
    """numpy float32 emulation of gelu_sig: clamp, two fmas, ex2.approx (exact exp2 rounded to fp32), 1 + e and the
    quotient in fp32."""
    x = np.asarray(x, F32)
    c4, c2, c0 = (np.float64(F32(c)) for c in coef)
    xc = np.clip(x, F32(-10), F32(10))
    x2 = (xc * xc).astype(F32)
    inner = (x2.astype(np.float64) * c4 + c2).astype(F32)
    pl = (x2.astype(np.float64) * inner.astype(np.float64) + c0).astype(F32)
    arg = (xc * pl).astype(F32)
    e = np.exp2(arg.astype(np.float64)).astype(F32)
    return (x / (F32(1) + e)).astype(F32)


def geglu_gate_errors(out_gate, g):
    """out_gate: fp16 fp16(gelu_sig(g)) (the v = 1 column), g: the fp16 pre-activations -> err / bound (float64).
    Bound: half an ulp of the result (the one fp16 rounding; at a binade edge the wider ulp) plus gelu_sig_bound."""
    out = out_gate.double()
    ref = gelu64(g)
    half_ulp = 0.5 * torch.maximum(ulp16(out), ulp16(ref))
    return (out - ref).abs() / (half_ulp + gelu_sig_bound(g))


def all_finite_f16() -> torch.Tensor:
    """The 63 488 finite fp16 values (both zeros included), ascending by bit pattern per sign."""
    b = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.float16)
    return b[torch.isfinite(b)]


# ------------------------------------------------------------------------------------------------- Swin windows
def padded(H, W, ws):
    return -(-H // ws) * ws, -(-W // ws) * ws


def window_gather_ref(x: torch.Tensor, ws: int, shift: int) -> torch.Tensor:
    """swin.py:269-287: zero-pad H, W to multiples of ws, roll by -shift, partition -> [B * nW, ws * ws, C]."""
    B, H, W, C = x.shape
    Hp, Wp = padded(H, W, ws)
    xp = F.pad(x, (0, 0, 0, Wp - W, 0, Hp - H))
    if shift:
        xp = torch.roll(xp, (-shift, -shift), (1, 2))
    return xp.reshape(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)


def window_scatter_ref(win: torch.Tensor, B: int, H: int, W: int, ws: int, shift: int) -> torch.Tensor:
    """swin.py:289-304: window reverse, roll by +shift, crop to [B, H, W, C]."""
    C = win.shape[-1]
    Hp, Wp = padded(H, W, ws)
    x = win.reshape(B, Hp // ws, Wp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, C)
    if shift:
        x = torch.roll(x, (shift, shift), (1, 2))
    return x[:, :H, :W]


def window_gather_index(B, H, W, ws, shift, mutant=None):
    """The gather kernel's map: for each output token (b, window, t) the flat source pixel b*H*W + sy*W + sx, or -1
    for a pad token.  mutant 'no_wrap': without the % Hp / % Wp wrap."""
    Hp, Wp = padded(H, W, ws)
    nWh, nWw = Hp // ws, Wp // ws
    b, wy, wx, t = np.meshgrid(np.arange(B), np.arange(nWh), np.arange(nWw), np.arange(ws * ws), indexing="ij")
    sy = wy * ws + t // ws + shift
    sx = wx * ws + t % ws + shift
    if mutant != "no_wrap":
        sy, sx = sy % Hp, sx % Wp
    src = (b * H + sy) * W + sx
    return np.where((sy < H) & (sx < W), src, -1).reshape(-1)


def window_scatter_index(B, H, W, ws, shift, mutant=None):
    """The scatter kernel's map: for each output pixel (b, y, x) the flat window token it reads.  mutant
    'shift_sign': the shift applied with the wrong sign."""
    Hp, Wp = padded(H, W, ws)
    nWh, nWw = Hp // ws, Wp // ws
    b, y, x = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), indexing="ij")
    s = -shift if mutant == "shift_sign" else shift
    sy, sx = (y - s + Hp) % Hp, (x - s + Wp) % Wp
    return ((((b * nWh + sy // ws) * nWw + sx // ws) * ws * ws) + (sy % ws) * ws + sx % ws).reshape(-1)


def apply_gather_index(x: torch.Tensor, idx, ws: int) -> torch.Tensor:
    B, H, W, C = x.shape
    flat = torch.cat([x.reshape(-1, C), torch.zeros(1, C, dtype=x.dtype)])
    idx = torch.as_tensor(idx)
    return flat[torch.where(idx < 0, flat.shape[0] - 1, idx)].reshape(-1, ws * ws, C)


def apply_scatter_index(win: torch.Tensor, idx, B, H, W) -> torch.Tensor:
    C = win.shape[-1]
    return win.reshape(-1, C)[torch.as_tensor(idx)].reshape(B, H, W, C)


# SeeCoder's Swin (configs.py: window 12, embed 192, four levels; 7 is the class default): the levels' grids at 512
# and 768 pixel inputs (patch 4), with the level's channel count, plus a grid smaller than a window and a ragged one
WINDOW_GEOMETRIES = [(128, 128, 192), (192, 192, 192), (64, 64, 384), (96, 96, 384), (32, 32, 768), (48, 48, 768),
                     (16, 16, 1536), (24, 24, 1536), (8, 8, 192), (13, 29, 384)]
WINDOW_SIZES = (12, 7)
