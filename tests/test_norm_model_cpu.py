"""CPU model of the GroupNorm and LayerNorm kernels (pfd_b200/csrc/elementwise.cu): shows that the float64 checks of
test_norm_gpu.py accept the kernels' arithmetic, reject the one-pass statistics without a pivot at large activation
offsets, and reject subtly wrong variants of the kernels.

The numpy emulator follows the kernels: the thread layout and pixel chunking of pfd_groupnorm_f16 (fast path with
plan_sms = 132, and the deterministic path), each thread's sequential fp32 sums of d = x - K_g and d^2 (fused) over its
pixels, the fp32 shared-memory fold of the fast path in thread order, fp64 across CTAs; the apply kernel's fp32 a, b
and fma with the fp16 value before SiLU; LayerNorm's lane-sequential fp32 sums, fp32 butterfly and fp16(x + residual).  The CPU cases are the GPU cases with HW capped at 4096 and NB at 2 (NB = 64 kept).
"""
import numpy as np
import pytest
import torch

from norm_ref import (GN_KINDS, GROUPS, LN_KINDS, RMS_LIMIT, gn_inputs, groupnorm_ref, layernorm_ref, ln_inputs,
                      norm_errors)
from test_norm_gpu import GN_SHAPES, LN_CHANNELS, ln_eps

PLAN_SMS = 132
F32, F64 = np.float32, np.float64
GN_MUTANTS = ("neighbour_group", "drop_tail", "eps_after_sqrt", "no_presilu_round")


def gn_layout(C, HW, NB, det):
    """(threads, pixel lanes, pixels per CTA, chunks) of pfd_groupnorm_f16."""
    vecs = C // 8
    threads = (256 // vecs) * vecs if vecs <= 256 else (vecs if vecs <= 320 else 256)
    if threads < 64:
        threads = vecs * (-(-64 // vecs))
    lanes = threads // vecs
    if det:
        ppc = -(-HW // 128)
    else:
        c0 = -(-3 * PLAN_SMS // NB)
        ppc = -(-HW // c0)
    ppc = max(ppc, 16 * max(lanes, 1))
    return threads, lanes, ppc, -(-HW // ppc)


def thread_sums(d, lanes, ppc, chunks, drop_tail=False):
    """d [HW, C] fp32 -> per-thread sequential fp32 sums of d and d^2 (fused), [chunks, lanes, C]; thread (chunk, lane)
    walks pixels chunk * ppc + lane + j * lanes.  drop_tail: skip the pixels after the last full group of 4."""
    HW, C = d.shape
    steps = -(-ppc // lanes)
    t = np.zeros((chunks, steps * lanes, C), F32)
    pad = np.zeros((chunks * ppc, C), F32)
    pad[:HW] = d
    t[:, :ppc] = pad.reshape(chunks, ppc, C)
    t = t.reshape(chunks, steps, lanes, C)
    if drop_tail:
        npix = np.minimum(ppc, HW - np.arange(chunks) * ppc)                  # pixels of each chunk
        per_lane = -(-(npix[:, None] - np.arange(lanes)[None, :]) // lanes)    # pixels of each (chunk, lane)
        full = (per_lane // 4) * 4
        keep = np.arange(steps)[None, :, None] < full[:, None, :]
        t = t * keep[..., None]
    sm = np.zeros((chunks, lanes, C), F32)
    sq = np.zeros((chunks, lanes, C), F32)
    for j in range(steps):
        tj = t[:, j]
        sm = (sm + tj).astype(F32)
        sq = (sq.astype(F64) + tj.astype(F64) ** 2).astype(F32)
    return sm, sq


def gn_stats(x, NB, HW, C, det, pivot=True, mutant=None):
    """x [NB, HW, C] fp32 (fp16 values) -> (S, Q, K) per (image, group): fp64 sums of d = x - K and d^2, the pivots."""
    cpg = C // GROUPS
    vecs = C // 8
    threads, lanes, ppc, chunks = gn_layout(C, HW, NB, det)
    gmap = np.arange(C) // cpg
    if mutant == "neighbour_group":
        gmap[cpg] = 0                          # the first channel of group 1 counted in group 0
    K = x[:, 0, np.arange(GROUPS) * cpg] if pivot else np.zeros((NB, GROUPS), F32)
    S = np.zeros((NB, GROUPS))
    Q = np.zeros((NB, GROUPS))
    for n in range(NB):
        d = (x[n] - K[n][gmap]).astype(F32)
        if det:
            # per-thread fp32 sums (a wide-row thread walks its chunk vector by vector), then fp64 folds
            sm, sq = thread_sums(d, max(lanes, 1), ppc, chunks, mutant == "drop_tail" and lanes >= 1)
            for s_out, part in ((S, sm), (Q, sq)):
                s_out[n] = np.bincount(np.tile(gmap, part.shape[0] * part.shape[1]),
                                       part.astype(F64).reshape(-1), GROUPS)
        else:
            # per-thread fp32 sums (a wide-row thread walks its chunk vector by vector); each thread folds its 8
            # channels into group bins (fp32, channel order), then the shared fp32 atomics in thread order
            lt = max(lanes, 1)
            sm, sq = thread_sums(d, lt, ppc, chunks, mutant == "drop_tail" and lanes >= 1)
            v = np.arange(vecs)
            for s_out, part in ((S, sm), (Q, sq)):
                bins = np.zeros((chunks, lt, vecs, GROUPS), F32)
                for i in range(8):
                    bins[:, :, v, gmap[v * 8 + i]] = (bins[:, :, v, gmap[v * 8 + i]] + part[:, :, v * 8 + i]).astype(F32)
                shared = np.cumsum(bins.reshape(chunks, lt * vecs, GROUPS), axis=1, dtype=F32)[:, -1]
                s_out[n] = shared.astype(F64).sum(0)
    return S, Q, K.astype(F64)


def gn_emulate(x1, x2, gamma, beta, eps, silu, det, pivot=True, mutant=None):
    """The kernels' output (fp16 torch [NB, HW, C]) for fp16 torch inputs."""
    x = (x1 if x2 is None else torch.cat([x1, x2], -1)).float().numpy()
    NB, HW, C = x.shape
    cpg = C // GROUPS
    S, Q, K = gn_stats(x, NB, HW, C, det, pivot, mutant)
    inv = 1.0 / (HW * cpg)
    m = S * inv
    var = np.maximum(Q * inv - m * m, 0.0)
    mean = (K + m).astype(F32)
    e32 = F32(eps)
    if mutant == "eps_after_sqrt":
        rstd = (1.0 / (np.sqrt(var.astype(F32).astype(F64)) + F64(e32))).astype(F32)
    else:
        rstd = (1.0 / np.sqrt((var.astype(F32) + e32).astype(F64))).astype(F32)
    gc = np.arange(C) // cpg
    ga, be = gamma.float().numpy(), beta.float().numpy()
    a = (rstd[:, None, gc] * ga).astype(F32)
    b = (be.astype(F64) - mean[:, None, gc].astype(F64) * a).astype(F32)
    y = (x.astype(F64) * a + b).astype(F32)
    if silu:
        z = y if mutant == "no_presilu_round" else y.astype(np.float16).astype(F32)
        with np.errstate(over="ignore"):
            e = np.exp(-z.astype(F64)).astype(F32)
            y = (z.astype(F64) / (1.0 + e.astype(F64)).astype(F32)).astype(F32)
    return torch.from_numpy(y.astype(np.float16))


def ln_emulate(x, res, gamma, beta, eps, mutant=None):
    """layernorm_kernel for fp16 torch inputs [rows, C] -> fp16 torch [rows, C]."""
    v = x.float().numpy()
    if res is not None:
        v = (v + res.float().numpy()).astype(F32)
        if mutant != "res_unrounded":
            v = v.astype(np.float16).astype(F32)
    rows, C = v.shape
    vecs = C // 8
    maxv = -(-vecs // 32)
    # lane l holds vectors l, l + 32, ...: element order k, then i
    lanes = np.zeros((rows, 32, maxv * 8), F32)
    for k in range(maxv):
        for ln in range(32):
            vi = ln + 32 * k
            if vi < vecs:
                lanes[:, ln, k * 8:(k + 1) * 8] = v[:, vi * 8:(vi + 1) * 8]
    valid = np.zeros((32, maxv * 8), bool)
    for k in range(maxv):
        valid[:min(32, max(0, vecs - 32 * k)), k * 8:(k + 1) * 8] = True

    def butterfly(t):
        for o in (16, 8, 4, 2, 1):
            t = (t + t[:, np.arange(32) ^ o]).astype(F32)
        return t[:, 0]

    s = butterfly(np.cumsum(lanes, axis=2, dtype=F32)[:, :, -1])
    mean = (s / F32(C)).astype(F32)
    d = np.where(valid, (lanes - mean[:, None, None]).astype(F32), F32(0))
    q = np.zeros((rows, 32), F32)
    for j in range(maxv * 8):
        q = (q.astype(F64) + d[:, :, j].astype(F64) ** 2).astype(F32)
    q = butterfly(q)
    rstd = (1.0 / np.sqrt(((q / F32(C)).astype(F32) + F32(eps)).astype(F64))).astype(F32)
    o = ((v - mean[:, None]).astype(F32) * rstd[:, None]).astype(F32)
    o = (o.astype(F64) * gamma.float().numpy() + beta.float().numpy()).astype(F32)
    return torch.from_numpy(o.astype(np.float16))


# ---------------------------------------------------------------------------------------------- CPU-sized cases
def cpu_gn_cases():
    for C1, C2, HW, NB, eps in GN_SHAPES:
        yield C1, C2, min(HW, 4096), (NB if NB == 64 else min(NB, 2)), eps


def gn_case_errors(case, kind, silu, det, pivot=True, mutant=None):
    C1, C2, HW, NB, eps = case
    x1, x2, gamma, beta, const = gn_inputs(NB, HW, C1, C2, kind)
    out = gn_emulate(x1, x2, gamma, beta, eps, silu, det, pivot, mutant)
    ref, bound, var = groupnorm_ref(x1, x2, gamma, beta, eps, silu)
    return norm_errors(out, ref, bound, var)


def gn_ids(c):
    return "C{}+{}-HW{}-NB{}".format(*c[:4])


@pytest.mark.parametrize("det", [False, True], ids=["fast", "det"])
@pytest.mark.parametrize("case", list(cpu_gn_cases()), ids=gn_ids)
def test_fixed_groupnorm_within_bound(case, det):
    """(a) the pivot-shifted statistics pass the bound and the rms check of every GPU case."""
    for kind in GN_KINDS:
        for silu in (False, True):
            worst, rms, nonfinite = gn_case_errors(case, kind, silu, det)
            assert nonfinite == 0 and worst <= 1.0 and rms <= RMS_LIMIT, (kind, silu, worst, rms, nonfinite)


@pytest.mark.parametrize("det", [False, True], ids=["fast", "det"])
def test_onepass_groupnorm_fails_large_offsets(det):
    """(b) the one-pass E[x^2] - mean^2 of unshifted fp32 sums fails the large-offset cases and passes the others."""
    failed = {}
    for case in cpu_gn_cases():
        if case[2] < 256:
            continue
        for kind in ("random", "dc16", "dc256", "dc1024"):
            worst, rms, nonfinite = gn_case_errors(case, kind, False, det, pivot=False)
            failed.setdefault(kind, []).append(bool(nonfinite) or worst > 1.0 or rms > RMS_LIMIT)
    print(f"[norm model] one-pass statistics, cases failed per kind: "
          f"{ {k: f'{sum(v)}/{len(v)}' for k, v in failed.items()} }")
    assert not any(failed["random"])
    assert all(failed["dc256"])
    assert all(failed["dc1024"])


def gn_rejected_by(mutant):
    caught = []
    for case in cpu_gn_cases():
        for kind in ("random", "dc16", "const"):
            for silu in (False, True):
                worst, rms, nonfinite = gn_case_errors(case, kind, silu, False, mutant=mutant)
                if nonfinite or worst > 1.0 or rms > RMS_LIMIT:
                    caught.append(f"{gn_ids(case)} {kind} silu={silu} (err/bound {worst:.3g}, rms {rms:.3g})")
    return caught


@pytest.mark.parametrize("mutant", GN_MUTANTS)
def test_groupnorm_mutant_rejected(mutant):
    """(c) the checks reject subtly wrong GroupNorm kernels."""
    caught = gn_rejected_by(mutant)
    print(f"[norm model] mutant {mutant}: rejected by {len(caught)} checks, first: {caught[0] if caught else 'none'}")
    assert caught, f"mutant {mutant} passes every check"


def ln_case_errors(C, rows, kind, residual, mutant=None):
    x, res, gamma, beta, _ = ln_inputs(rows, C, kind)
    r = res if residual else None
    out = ln_emulate(x, r, gamma, beta, ln_eps(kind), mutant)
    ref, bound, var = layernorm_ref(x, r, gamma, beta, ln_eps(kind))
    return norm_errors(out, ref, bound, var)


@pytest.mark.parametrize("C", LN_CHANNELS)
def test_layernorm_within_bound(C):
    """(a) the LayerNorm arithmetic passes the bound and the rms check of every GPU case."""
    for kind in LN_KINDS:
        for residual in (False, True):
            worst, rms, nonfinite = ln_case_errors(C, 200, kind, residual)
            assert nonfinite == 0 and worst <= 1.0 and rms <= RMS_LIMIT, (kind, residual, worst, rms, nonfinite)


def test_layernorm_mutant_rejected():
    """(c) the checks reject a LayerNorm that does not round x + residual to fp16."""
    caught = []
    for C in LN_CHANNELS:
        for kind in ("random", "dc16"):
            worst, rms, nonfinite = ln_case_errors(C, 200, kind, True, "res_unrounded")
            if nonfinite or worst > 1.0 or rms > RMS_LIMIT:
                caught.append(f"C{C} {kind} (err/bound {worst:.3g}, rms {rms:.3g})")
    print(f"[norm model] mutant res_unrounded: rejected by {len(caught)} checks, first: "
          f"{caught[0] if caught else 'none'}")
    assert caught
