"""CPU model of the flash-attention kernel (pfd_b200/csrc/attention.cu): shows that the float64 checks of
test_attention_gpu.py accept the kernel's algorithm and reject subtly wrong variants of it.

The numpy emulator follows the kernel: 64-key blocks, fp32 logits, p = 2^(s c2 - m) against the running max and
rounded to fp16, the row sum l taken from the rounded p, o and l rescaled by alpha = 2^(m_old - m_new) when the max
moves, keys past Nk read as TMA zero fill and masked to -inf, one fp16 rounding of o / l.
"""
import numpy as np
import pytest
import torch

from attention_ref import (BKV, HEAD_DIM_CASES, RETRIEVAL_CASES, ROW_MAX_CASES, TILE_EDGE_CASES, c2_of, flash_errors,
                           flash_inputs, retrieval_inputs, RMS_LIMIT)

MUTANTS = ("ghost_key", "no_o_rescale", "drop_last_block", "drop_last_8_channels")


def emulate(q, k, v, scale, mutant=None):
    """q [Nq, d], k / v [Nk, d] fp16 numpy arrays -> O [Nq, d] fp16."""
    Nq, d = q.shape
    Nk = k.shape[0]
    nblk = -(-Nk // BKV)
    c2 = np.float32(c2_of(scale))
    kz = np.zeros((nblk * BKV, d), np.float32)         # TMA zero fill past Nk
    vz = np.zeros((nblk * BKV, d), np.float32)
    kz[:Nk], vz[:Nk] = k, v
    if mutant == "drop_last_8_channels" and d % 16 == 8:
        kz[:, d - 8:] = 0
    qf = q.astype(np.float32)
    m = np.full(Nq, -np.inf, np.float32)
    l = np.zeros(Nq, np.float32)
    o = np.zeros((Nq, d), np.float32)
    blocks = range(Nk // BKV if mutant == "drop_last_block" and Nk % BKV else nblk)
    for j in blocks:
        s = qf @ kz[j * BKV:(j + 1) * BKV].T
        valid = Nk - j * BKV + (mutant == "ghost_key")
        s[:, max(valid, 0):] = -np.inf
        mnew = np.maximum(m, (s.max(1) * c2).astype(np.float32))
        with np.errstate(invalid="ignore"):
            alpha = np.exp2((m - mnew).astype(np.float64)).astype(np.float32)
        alpha = np.where(np.isneginf(m), np.float32(0), alpha)
        m = mnew
        l *= alpha
        if mutant != "no_o_rescale":
            o *= alpha[:, None]
        t = (s.astype(np.float64) * np.float64(c2) - m[:, None]).astype(np.float32)     # one fma rounding
        p = np.exp2(t.astype(np.float64)).astype(np.float32).astype(np.float16).astype(np.float32)
        l += p.sum(1, dtype=np.float32)
        o += p @ vz[j * BKV:(j + 1) * BKV]
    inv = np.where(l > 0, np.float32(1) / np.where(l > 0, l, 1), np.float32(0)).astype(np.float32)
    return (o * inv[:, None]).astype(np.float16)


def run(q, k, v, scale, mutant=None):
    return torch.from_numpy(np.stack([emulate(q[g].numpy(), k[g].numpy(), v[g].numpy(), scale, mutant)
                                      for g in range(q.shape[0])]))


def scaled(case, qmax=48):
    """A GPU case cut to one (batch, head) and at most qmax query rows (rows are independent); Nk and d stay."""
    B, heads, Nq, Nk, d, kind = case
    q, k, v, scale = flash_inputs(B, heads, Nq, Nk, d, kind)
    return q[:1, :qmax], k[:1], v[:1], scale


@pytest.mark.parametrize("case", HEAD_DIM_CASES + TILE_EDGE_CASES + ROW_MAX_CASES,
                         ids=lambda c: "B{}h{}q{}k{}d{}-{}".format(*c))
def test_emulator_within_bound(case):
    q, k, v, scale = scaled(case)
    worst, rms, nonfinite = flash_errors(run(q, k, v, scale), q, k, v, scale)
    assert nonfinite == 0 and worst <= 1.0 and rms <= RMS_LIMIT, (worst, rms, nonfinite)


@pytest.mark.parametrize("case", RETRIEVAL_CASES, ids=lambda c: "B{}h{}q{}k{}d{}{}".format(*c[:5], "-ghost" * c[5]))
def test_emulator_exact_retrieval(case):
    q, k, v, expect = retrieval_inputs(*case)
    assert torch.equal(run(q, k, v, 1.0), expect)


def rejected_by(mutant):
    """Names of the GPU file's checks that reject the mutant (scaled-down cases run on the emulator)."""
    caught = []
    for case in HEAD_DIM_CASES + TILE_EDGE_CASES + ROW_MAX_CASES:
        q, k, v, scale = scaled(case, qmax=16)
        worst, rms, nonfinite = flash_errors(run(q, k, v, scale, mutant), q, k, v, scale)
        if nonfinite or worst > 1.0:
            caught.append(f"bound {case} (err/bound {worst:.3g})")
        if rms > RMS_LIMIT:
            caught.append(f"rms {case} (rms ratio {rms:.3g})")
    for case in RETRIEVAL_CASES:
        q, k, v, expect = retrieval_inputs(*case)
        if not torch.equal(run(q, k, v, 1.0, mutant), expect):
            caught.append(f"exact retrieval {case}")
    return caught


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_rejected(mutant):
    caught = rejected_by(mutant)
    print(f"[attention model] mutant {mutant}: rejected by {len(caught)} checks, first: "
          f"{caught[0] if caught else 'none'}")
    assert caught, f"mutant {mutant} passes every check"
