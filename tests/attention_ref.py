"""Float64 references, error bounds and input generators for the attention tests (test_attention_gpu.py and its CPU
model test_attention_model_cpu.py).  This module holds no tests.

Flash attention (pfd_b200/csrc/attention.cu) computes O = softmax(scale Q K^T) V with fp32 logits, p = fp16(2^(t - m))
against the running row max m (t = logit in log2 units), fp32 rescales of o and l when m moves, the row sum l taken
from the rounded p, and one final fp16 rounding.  ``flash_errors`` compares an output against the exact float64 result
with a per-element worst-case bound derived from those rounding points, and against a model of the random part of the
error (an rms check, which catches a systematic bias that the worst-case bound would absorb).

The softmax kernel (pfd_b200/csrc/elementwise.cu, unfused attention path) keeps the reference's fp16 rounding points:
rh(rh(x * scale) + bias) + mask, then an fp32 softmax rounded to fp16.
"""
import math

import numpy as np
import torch

LOG2E = 1.4426950408889634
BKV = 64                     # keys per block of the flash kernel
K_BOUND = 1.25               # safety factor of the worst-case bound over its first-order terms
RMS_LIMIT = 3.0              # rms(err) / rms(model sigma) limit


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |x| (float64); 2^-24 in the subnormal range and at 0."""
    _, e = torch.frexp(x.abs().double())               # frexp(0) has exponent 0: clamp it to the subnormal one
    e = torch.where(x == 0, torch.full_like(e, -13), e)
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 11).clamp_min(2.0 ** -24)


def rh(x: torch.Tensor) -> torch.Tensor:
    """fp32 value rounded to fp16, as float64 (the kernels' __float2half_rn)."""
    return x.float().half().double()


def c2_of(scale: float) -> float:
    """The kernel's fp32 constant scale * log2(e)."""
    return float(np.float32(scale) * np.float32(LOG2E))


def flash_ref_one(q, k, v, scale):
    """One (batch, head): q [Nq, d], k / v [Nk, d] (fp16 values) -> (O, bound, sigma^2), float64 [Nq, d]."""
    Q, Kd, V = q.double(), k.double(), v.double()
    Nk, d = Kd.shape
    nblk = -(-Nk // BKV)
    t = (Q @ Kd.T) * (float(np.float32(scale)) * LOG2E)        # exact logits, log2 units
    M = t.amax(1, keepdim=True)
    e = torch.exp2(t - M)
    L = e.sum(1, keepdim=True)
    w = e / L
    O = w @ V
    Va, Oa = V.abs(), O.abs()
    # relative error of each p: fp16 rounding, ex2.approx, fp32 logit accumulation (d products), the fp32 c2 and the
    # fp32 rounding of t - m
    eps = 2.0 ** -11 + 2.0 ** -21 + math.log(2) * (c2_of(scale) * d * 2.0 ** -24 * (Q.abs() @ Kd.abs().T)
                                                   + (t.abs() + M.abs()) * 2.0 ** -23)
    we = w * (eps + eps.amax(1, keepdim=True))
    del eps, t, e
    bound = we @ Va + we.sum(1, keepdim=True) * Oa                          # sum_j w_j (eps_j + eps_max)(|v| + |O|)
    bound += (2 * 2.0 ** -25) / L * (Va.sum(0, keepdim=True) + Nk * Oa)    # p flushed / subnormal in fp16
    bound += (2 * nblk + 64) * 2.0 ** -24 * (w @ Va)                        # fp32 accumulation and rescales
    bound = K_BOUND * bound + ulp16(O)
    w2 = w * w
    var = (w2 @ (V * V) - 2 * O * (w2 @ V) + O * O * w2.sum(1, keepdim=True)).clamp_min(0) * (2.0 ** -22 / 3)
    var += ulp16(O) ** 2 / 12
    return O, bound, var


def flash_errors(out, q, k, v, scale):
    """out, q [G, Nq, d], k / v [G, Nk, d] -> (largest err / bound, rms(err) / rms(sigma), number of non-finite
    outputs).  One (batch, head) at a time to bound the memory of the [Nq, Nk] float64 weights."""
    worst, se, sv = 0.0, 0.0, 0.0
    nonfinite = int((~torch.isfinite(out)).sum())
    if nonfinite:
        return math.inf, math.inf, nonfinite
    for g in range(q.shape[0]):
        O, bound, var = flash_ref_one(q[g], k[g], v[g], scale)
        err = (out[g].double() - O).abs()
        worst = max(worst, float((err / bound).max()))
        se += float((err * err).sum())
        sv += float(var.sum())
    return worst, math.sqrt(se / sv), 0


def flash_check(out, q, k, v, scale, label):
    """Assert the bound and the rms check; prints both ratios."""
    worst, rms, nonfinite = flash_errors(out, q, k, v, scale)
    print(f"[attention f64] {label}: max err/bound {worst:.3f}, rms err/sigma {rms:.3f}")
    assert nonfinite == 0, f"{label}: {nonfinite} non-finite outputs"
    assert worst <= 1.0, f"{label}: error exceeds the bound by {worst:.3f}x"
    assert rms <= RMS_LIMIT, f"{label}: rms error {rms:.3f}x the model sigma"


# ---------------------------------------------------------------------------------------------- flash test cases
# (B, heads, Nq, Nk, d, kind); every case runs through both entry points on the GPU and through the emulator on the CPU
HEAD_DIM_CASES = [(2, 3, 130, 77, d, "random") for d in range(8, 193, 8)]
TILE_EDGE_CASES = ([(1, 2, nq, 77, d, "random") for nq in (1, 127, 128, 129, 257) for d in (40, 72, 160)]
                   + [(1, 2, 130, nk, d, "random") for nk in (1, 7, 8, 63, 64, 65, 128, 129, 192, 193, 4097)
                      for d in (40, 72, 160)])
ROW_MAX_CASES = [(1, 2, 130, nk, d, kind) for kind in ("increasing", "decreasing", "last_block_max", "constant", "huge")
                 for nk, d in ((1000, 64), (193, 72))]


def flash_inputs(B, heads, Nq, Nk, d, kind, seed=0):
    """q [B*heads, Nq, d], k / v [B*heads, Nk, d] fp16 CPU tensors and the softmax scale of one case.
    kind: 'random' (unit normal), 'increasing' / 'decreasing' (logits run monotonically along the keys from -17 to
    +17 log2 units, so the running max moves in every block or never), 'last_block_max' (the row max lies in the
    ragged last block), 'constant' (q = 0: O is the mean of V), 'huge' (|logits| ~ 10^3 in log2 units)."""
    G = B * heads
    g = torch.Generator().manual_seed(seed * 7919 + Nq * 131 + Nk * 17 + d)
    q = torch.randn((G, Nq, d), generator=g)
    k = torch.randn((G, Nk, d), generator=g)
    v = torch.randn((G, Nk, d), generator=g)
    scale = d ** -0.5
    if kind in ("increasing", "decreasing"):
        # channel 0 carries the trend: scale q_0 k_0 = 4 * ramp runs over +-12 natural units (+-17 log2 units); the
        # other channels add noise of ~0.5 natural units
        ramp = torch.linspace(-3.0, 3.0, Nk) * (1 if kind == "increasing" else -1)
        q[..., 0] = 4.0 * math.sqrt(d)
        k[..., 0] = ramp
        q[..., 1:] *= 0.5
    elif kind == "last_block_max":
        q[..., 0] = 3.0              # the last key's logit is ~12 natural (~17 log2) units above the others for every query
        k[:, Nk - 1, 0] = 4.0 * math.sqrt(d)
    elif kind == "constant":
        q.zero_()
    elif kind == "huge":
        q *= 24.0
        k *= 24.0
    elif kind != "random":
        raise ValueError(kind)
    return q.half(), k.half(), v.half(), scale


# ---------------------------------------------------------------------------------------------- exact retrieval
RETRIEVAL_A = 14             # |q| per code channel: non-target logits sit >= 2 A log2(e) = 40.4 log2 units lower
RETRIEVAL_CASES = [(2, 3, 130, 100, 8, False), (2, 3, 257, 4097, 40, False), (1, 2, 130, 1000, 72, False),
                   (2, 3, 130, 193, 136, False), (1, 2, 130, 129, 192, False),
                   (2, 3, 130, 63, 8, True), (1, 2, 130, 1000, 72, True), (2, 3, 130, 77, 160, True)]


def retrieval_inputs(B, heads, Nq, Nk, d, ghost):
    """Attention that retrieves one V row per query exactly (scale = 1).

    Each key of a (batch, head) gets a distinct +-1 code (its low channels hold a per-head permutation of the key
    index in binary, the others are random signs); query i is RETRIEVAL_A * code of key sigma(i), so its target logit
    beats every other key by >= 40 log2 units: every other p rounds to 0 in fp16 and the target's to 1, and O_i is
    V row sigma(i) bit for bit.  V rows are distinct nonzero integers <= 1021 that depend on (batch, head, key); sigma
    covers key 0, the first and last key of every 64-key block, and the last key.
    ghost: channel d-1 is a bias channel (q = -(A (d-1) + 28), k = 1 for real keys) that puts every real logit >= 40
    log2 units below 0, the logit of a zero-filled key past Nk, so a kernel that let one in would output a zero row.
    Returns q [G, Nq, d], k / v [G, Nk, d] (fp16) and the expected output [G, Nq, d]."""
    G = B * heads
    dc = d - 1 if ghost else d
    assert Nk <= 2 ** (dc - 1), "codes must be distinct"
    nb = max(1, (Nk - 1).bit_length())
    gen = torch.Generator().manual_seed(Nk * 1000 + d + ghost)
    special = sorted({0, Nk - 1} | {j for b0 in range(0, Nk, BKV) for j in (b0, min(b0 + BKV - 1, Nk - 1))})
    assert len(special) <= Nq
    q = torch.zeros((G, Nq, d))
    k = torch.zeros((G, Nk, d))
    v = torch.zeros((G, Nk, d))
    expect = torch.zeros((G, Nq, d))
    bits = 2 ** torch.arange(nb)
    for gi in range(G):
        perm = torch.randperm(Nk, generator=gen)
        code = torch.where(torch.randint(0, 2, (Nk, dc), generator=gen) == 1, 1.0, -1.0)
        code[:, :nb] = torch.where((perm[:, None] & bits) != 0, 1.0, -1.0)
        k[gi, :, :dc] = code
        idx = (gi * Nk + torch.arange(Nk))[:, None]
        c = torch.arange(d)[None, :]
        v[gi] = (1 + (idx * (c + 1) + 13 * c) % (1021 - 2 * c)) * (1 - 2 * (c % 2))
        sigma = torch.cat([torch.tensor(special), torch.randint(0, Nk, (Nq - len(special),), generator=gen)])
        sigma = sigma[torch.randperm(Nq, generator=gen)]
        q[gi, :, :dc] = RETRIEVAL_A * code[sigma]
        expect[gi] = v[gi, sigma]
    if ghost:
        q[..., d - 1] = -(RETRIEVAL_A * dc + 28)
        k[..., d - 1] = 1.0
    return q.half(), k.half(), v.half(), expect.half()


# ---------------------------------------------------------------------------------------------- softmax kernel
def softmax_ref(x, scale, bias=None, mask=None):
    """Float64 softmax of rows with the kernel's rounding points rh(rh(rh(x * scale) + bias) + mask).
    Returns (probabilities, the rounded logits)."""
    t = rh(x.double() * float(np.float32(scale)))
    if bias is not None:
        t = rh(t + bias.double())
    if mask is not None:
        t = rh(t + mask.double())
    p = torch.softmax(t, -1)
    return p, t


def softmax_bound(p, t):
    """One fp16 ulp plus the fp32 error of __expf, the row sum and the normalisation."""
    cols = t.shape[-1]
    gap = t.amax(-1, keepdim=True) - t
    return ulp16(p) + p * (2.0 ** -20 + gap * 2.0 ** -23 + cols * 2.0 ** -24)
