"""Float64 references, error bounds and input generators for the normalisation tests (test_norm_gpu.py and its CPU
model test_norm_model_cpu.py).  This module holds no tests.

GroupNorm (pfd_b200/csrc/elementwise.cu, gn_stats / gn_stats_det / gn_apply) reduces per-(image, group) sums of x and
x^2 (shifted by a per-group pivot) to fp64, then applies a = fp32(rstd * gamma), b = fp32(beta - mean * a),
y = fmaf(x, a, b) with rstd = rsqrtf(fp32(var) + eps), [z = fp16(y), y = __fdividef(z, 1 + __expf(-z))], and one fp16
rounding.  ``groupnorm_ref`` returns the exact float64 output with those rounding points (eps as fp32, the fp16 value
before SiLU), a per-element worst-case bound built from the apply arithmetic plus a fixed budget STATS_REL for the
statistics, and a model of the random part of the error for an rms check (which catches a systematic bias that the
worst-case bound would absorb).  No term of the bound grows with (mean / std)^2: a kernel whose statistics lose
precision to a large common offset of the activations fails it.

LayerNorm (layernorm_kernel) rounds x + residual to fp16, takes the mean and then the centred sum of squares of the
row in fp32 (one warp per row, lane-sequential sums and a 32-lane butterfly), and outputs fp16(((v - mean) * rstd) *
gamma + beta).  ``layernorm_ref`` bounds each term of that arithmetic in the worst case.
"""
import math

import numpy as np
import torch

from attention_ref import rh, ulp16

GROUPS = 32
K_BOUND = 1.25               # safety factor of the worst-case bounds over their first-order terms
RMS_LIMIT = 3.0              # rms(err) / rms(model sigma) limit
STATS_REL = 2.0 ** -17       # statistics budget: relative error of rstd, and error of the mean in units of std
U32 = 2.0 ** -24             # fp32 unit roundoff
RSQRT_REL = 2.0 ** -22       # rsqrtf: at most 2 fp32 ulps
SILU_DERIV_MAX = 1.1         # max |d silu / dz|


def _silu_kernel_rel(z):
    """Relative error of __fdividef(z, 1 + __expf(-z)): __expf is within 2 + 1.173 |z| ulps, and its share of the
    denominator is e / (1 + e); the fp32 add and __fdividef (2 ulps)."""
    return torch.sigmoid(-z) * (2.0 + 1.173 * z.abs()) * 2.0 ** -23 + 5 * U32


def groupnorm_ref(x1, x2, gamma, beta, eps, silu):
    """x1 [NB, HW, C1], x2 [NB, HW, C2] or None (fp16, any device), gamma / beta [C] -> (out, bound, var), float64
    [NB, HW, C]: the exact output with the kernel's rounding points, the worst-case error bound and the model variance
    of the random error."""
    x = x1.double() if x2 is None else torch.cat([x1, x2], -1).double()
    NB, HW, C = x.shape
    cpg = C // GROUPS
    xg = x.reshape(NB, HW, GROUPS, cpg)
    mu = xg.mean((1, 3), keepdim=True)
    var = (xg - mu).pow(2).mean((1, 3), keepdim=True)
    r = 1.0 / torch.sqrt(var + float(np.float32(eps)))
    sd = var.sqrt()
    xc = (xg - mu).reshape(NB, HW, C)
    mu_c = mu.expand(NB, 1, GROUPS, cpg).reshape(NB, 1, C)
    sd_c = sd.expand(NB, 1, GROUPS, cpg).reshape(NB, 1, C)
    A = gamma.double().abs() * r.expand(NB, 1, GROUPS, cpg).reshape(NB, 1, C)
    y = xc * (A * gamma.double().sign()) + beta.double()
    b_abs = beta.double().abs() + A * mu_c.abs()
    # rstd (statistics, rsqrtf, fp32 var and + eps, the rounding of a) scales x - mean; the mean's budget, its fp32
    # cast and b = beta - mean * a shift every output of the channel; the fma rounds once
    e_pre = (A * xc.abs() * (STATS_REL + RSQRT_REL + 3 * U32) + A * sd_c * STATS_REL
             + U32 * (3 * A * mu_c.abs() + b_abs + y.abs()))
    e_pre = K_BOUND * e_pre
    v_pre = (U32 * (y.abs() + b_abs + 2 * A * mu_c.abs() + 2 * A * xc.abs())) ** 2 / 3
    if not silu:
        return y, e_pre + 0.5 * ulp16(y.abs() + e_pre), v_pre + ulp16(y) ** 2 / 12
    z = rh(y)
    dz = torch.maximum((rh(y + e_pre) - z).abs(), (rh(y - e_pre) - z).abs())
    s = z * torch.sigmoid(z)
    e_s = SILU_DERIV_MAX * dz + K_BOUND * (s.abs() + SILU_DERIV_MAX * dz) * _silu_kernel_rel(z)
    ds = torch.sigmoid(z) * (1 + z * torch.sigmoid(-z))
    var_s = ds ** 2 * v_pre + (s * _silu_kernel_rel(z)) ** 2 / 3 + ulp16(s) ** 2 / 12
    return s, e_s + 0.5 * ulp16(s.abs() + e_s), var_s


def layernorm_ref(x, res, gamma, beta, eps):
    """x, res [rows, C] (res may be None; fp16, any device), gamma / beta [C] -> (out, bound, var), float64 [rows, C].
    The input is rounded at the kernel's point v = fp16(x + res)."""
    v = x.double() if res is None else rh(x.double() + res.double())
    rows, C = v.shape
    nl = 8 * -(-(C // 8) // 32)              # terms of one lane's sequential sum
    mu = v.mean(1, keepdim=True)
    vc = v - mu
    var = vc.pow(2).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + float(np.float32(eps)))
    y = vc * r * gamma.double() + beta.double()
    G = gamma.double().abs()
    vabs = v.abs().mean(1, keepdim=True)
    # the fp32 row sum (nl sequential adds per lane, 5 butterfly levels) and the division by C
    dmu = (nl + 5) * U32 * vabs + U32 * mu.abs()
    # rstd: the centred fp32 sum of squares, / C, + eps, rsqrtf, and the mean error's second-order term
    rr = 0.5 * ((nl + 8) * U32 + dmu ** 2 / (var + float(np.float32(eps)))) + RSQRT_REL
    e_pre = G * r * (dmu + vc.abs() * (rr + 3 * U32)) + U32 * y.abs()
    e_pre = K_BOUND * e_pre
    v_pre = (G * r * U32 * vabs) ** 2 * (nl + 5) / 3 + (U32 * (y.abs() + G * r * vc.abs())) ** 2 / 3
    return y, e_pre + 0.5 * ulp16(y.abs() + e_pre), v_pre + ulp16(y) ** 2 / 12


def norm_errors(out, ref, bound, var):
    """-> (largest err / bound, rms(err) / rms(model sigma), number of non-finite outputs)."""
    nonfinite = int((~torch.isfinite(out)).sum())
    if nonfinite:
        return math.inf, math.inf, nonfinite
    err = (out.double() - ref).abs()
    worst = float((err / bound).max())
    rms = math.sqrt(float((err * err).sum()) / float(var.sum()))
    return worst, rms, 0


def norm_check(out, ref, bound, var, label):
    """Assert the bound and the rms check; prints both ratios."""
    worst, rms, nonfinite = norm_errors(out, ref, bound, var)
    print(f"[norm f64] {label}: max err/bound {worst:.3f}, rms err/sigma {rms:.3f}")
    assert nonfinite == 0, f"{label}: {nonfinite} non-finite outputs"
    assert worst <= 1.0, f"{label}: error exceeds the bound by {worst:.3f}x"
    assert rms <= RMS_LIMIT, f"{label}: rms error {rms:.3f}x the model sigma"


# ---------------------------------------------------------------------------------------------- inputs
# kind: 'random' (N(0.5, 2^2)), 'dc<r>' (a per-(image, group) offset of r std, random sign, std 1), 'chan256' (per-channel
# offsets of 256 +- 4 std inside each group), 'const' (every 4th group constant, the next one with std 2^-6, the rest
# random), 'outlier256' (offset 256 std, and pixel 0 of every channel 4 std off the group mean), 'affine' (gamma with
# zeros and negative values, beta ~ N(0, 64^2))
GN_KINDS = ("random", "dc0", "dc16", "dc256", "dc1024", "chan256", "const", "outlier256", "affine")
LN_KINDS = ("random", "dc16", "dc256", "dc1024", "const", "affine")


def _affine(C, kind, g):
    if kind == "affine":
        gamma = 2.0 * torch.randn(C, generator=g)
        gamma[::8] = 0.0
        beta = 64.0 * torch.randn(C, generator=g)
    else:
        gamma = 1.0 + 0.5 * torch.randn(C, generator=g)
        gamma[5::16] = 0.0
        gamma[11::16] *= -1.0
        beta = 0.5 * torch.randn(C, generator=g)
    return gamma.half(), beta.half()


def gn_inputs(NB, HW, C1, C2, kind, seed=0):
    """x1 [NB, HW, C1], x2 [NB, HW, C2] or None, gamma, beta [C] (fp16, CPU) of one GroupNorm case, and the float
    mask [C] of the constant groups (all zero but for kind 'const')."""
    C = C1 + C2
    cpg = C // GROUPS
    g = torch.Generator().manual_seed(seed * 7919 + NB * 1009 + HW * 31 + C1 * 3 + C2 + GN_KINDS.index(kind))
    x = torch.randn((NB, HW, C), generator=g)
    const = torch.zeros(C)
    if kind == "random":
        x = 2.0 * x + 0.5
    elif kind.startswith("dc"):
        ratio = float(kind[2:])
        sign = torch.where(torch.rand((NB, 1, GROUPS, 1), generator=g) < 0.5, -1.0, 1.0)
        x = (x.reshape(NB, HW, GROUPS, cpg) + ratio * sign).reshape(NB, HW, C)
    elif kind == "chan256":
        x = x + 256.0 + 4.0 * torch.randn((NB, 1, C), generator=g)
    elif kind == "outlier256":
        sign = torch.where(torch.rand((NB, 1, GROUPS, 1), generator=g) < 0.5, -1.0, 1.0)
        xg = x.reshape(NB, HW, GROUPS, cpg)
        xg[:, 0] = 4.0 * sign[:, 0]
        x = (xg + 256.0 * sign).reshape(NB, HW, C)
    elif kind == "const":
        xg = x.reshape(NB, HW, GROUPS, cpg)
        level = torch.linspace(-2.0, 2.0, GROUPS)
        xg[:, :, 0::4] = level[0::4, None]
        xg[:, :, 1::4] = level[1::4, None] + 2.0 ** -6 * xg[:, :, 1::4]
        const.reshape(GROUPS, cpg)[0::4] = 1.0
    elif kind != "affine":
        raise ValueError(kind)
    gamma, beta = _affine(C, kind, g)
    x = x.half()
    return x[..., :C1].contiguous(), (x[..., C1:].contiguous() if C2 else None), gamma, beta, const


def ln_inputs(rows, C, kind, seed=0):
    """x, res [rows, C], gamma, beta [C] (fp16, CPU) of one LayerNorm case and the float mask [rows] of the constant
    rows (all zero but for kind 'const', where every 3rd row of x and res is constant)."""
    g = torch.Generator().manual_seed(seed * 7919 + rows * 131 + C * 7 + LN_KINDS.index(kind))
    x = torch.randn((rows, C), generator=g)
    res = torch.randn((rows, C), generator=g)
    const = torch.zeros(rows)
    if kind == "random":
        x = 2.0 * x + 0.3
    elif kind.startswith("dc"):
        ratio = float(kind[2:])
        x = x + ratio * torch.where(torch.rand((rows, 1), generator=g) < 0.5, -1.0, 1.0)
    elif kind == "const":
        x[0::3] = torch.linspace(-3.0, 3.0, rows)[0::3, None]
        res[0::3] = 0.25
        const[0::3] = 1.0
    elif kind != "affine":
        raise ValueError(kind)
    gamma, beta = _affine(C, kind, g)
    return x.half(), res.half(), gamma, beta, const
