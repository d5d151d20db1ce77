"""CPU model of the elementwise kernels the GPU tests check exactly (test_elementwise_gpu.py): shows that those checks
accept the kernels' arithmetic and reject subtly wrong variants of it.

* DDIM update: a numpy float32 emulation of ddim_step_kernel against the reference step in CPU torch fp16 (the same
  per-op fp32 compute and fp16 rounding as on the GPU), compared bit for bit over every schedule index.  Rejected
  variants: temperature rounded to fp16, guidance rounded to fp16, e_c - e_u left unrounded, and the dir_xt
  coefficient sqrt(1 - a_prev - sigma^2) without its intermediate fp16 roundings.
* GEGLU gate: a float32 emulation of gelu_sig over every finite fp16 input against the float64 bound of the GPU test;
  one coefficient off by 1e-3 relative is rejected.
* Swin window maps: the gather / scatter kernels' index arithmetic against the reference's pad -> roll -> partition
  views; scatter with the shift sign flipped and gather without the % Hp wrap are rejected.
"""
import numpy as np
import pytest
import torch

from elementwise_ref import (DDIM_GUIDANCE_CFG, DDIM_GUIDANCE_NOCFG, DDIM_MUTANTS, DDIM_STEPS, GELU_SIG_COEF,
                             WINDOW_GEOMETRIES, WINDOW_SIZES, all_finite_f16, apply_gather_index,
                             apply_scatter_index, bit_mismatch, bits, ddim_coefs, ddim_eager, ddim_inputs, ddim_kernel_model,
                             ddim_schedule_sampler, geglu_gate_errors, gelu64, gelu_sig_model, window_gather_index,
                             window_gather_ref, window_scatter_index, window_scatter_ref)


@pytest.fixture(scope="module")
def samplers():
    return {eta: ddim_schedule_sampler(eta) for eta in (0.0, 1.0)}


def ddim_mismatches(sampler, eps, x, noise, guidance, temperature, cfg, mutant=None):
    """(x_prev, pred_x0) mismatches of the kernel model against the eager fp16 reference, summed over every schedule
    index."""
    coef = sampler._coef_table()
    n_xp = n_p0 = 0
    for index in range(DDIM_STEPS):
        c = ddim_coefs(sampler, index, False, "cpu", x.dim())
        xp_r, p0_r = ddim_eager(eps, x, guidance, c, noise, temperature, cfg)
        xp_k, p0_k = ddim_kernel_model(eps.reshape(-1).numpy(), x.reshape(-1).numpy(), guidance, coef[index].tolist(),
                                       None if noise is None else noise.reshape(-1).numpy(), temperature, mutant)
        n_xp += int(bit_mismatch(xp_r, torch.from_numpy(xp_k)).sum())
        n_p0 += int(bit_mismatch(p0_r, torch.from_numpy(p0_k)).sum())
    return n_xp, n_p0


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("guidance", DDIM_GUIDANCE_CFG + DDIM_GUIDANCE_NOCFG)
def test_ddim_model_matches_eager_reference(samplers, eta, guidance):
    cfg = guidance not in DDIM_GUIDANCE_NOCFG
    for scale in (1.0, 30.0):
        eps, x, noise = ddim_inputs((2, 4, 13, 7), scale, seed=int(guidance * 10), cfg=cfg)
        for temperature in (1.0, 0.5, 0.7, 0.9):
            for nz in (noise, None):
                got = ddim_mismatches(samplers[eta], eps, x, nz, guidance, temperature, cfg)
                assert got == (0, 0), f"scale {scale} temperature {temperature} noise {nz is not None}: {got}"


@pytest.mark.parametrize("mutant", DDIM_MUTANTS)
def test_ddim_check_rejects_mutant(samplers, mutant):
    eps, x, noise = ddim_inputs((2, 4, 32, 32), 1.0, seed=3)
    guidance = 1.8 if mutant == "rh_guidance" else 7.5
    temperature = 0.7 if mutant == "rh_temperature" else 1.0
    n_xp, n_p0 = ddim_mismatches(samplers[1.0], eps, x, noise, guidance, temperature, True, mutant)
    print(f"[ddim mutant] {mutant}: {n_xp} x_prev / {n_p0} pred_x0 mismatches over {DDIM_STEPS} steps")
    assert n_xp > 0, f"{mutant} is not rejected"


def test_ddim_rh_temperature_only_matters_off_fp16(samplers):
    """The temperatures the sampling-loop tests use (1, 0.5) are fp16 values: rounding them changes nothing, which is
    why only 0.7 / 0.9 expose the rounded temperature."""
    eps, x, noise = ddim_inputs((2, 4, 13, 7), 1.0, seed=5)
    for t in (1.0, 0.5):
        assert ddim_mismatches(samplers[1.0], eps, x, noise, 7.5, t, True, "rh_temperature") == (0, 0)


def test_coef_table_rounds_like_torch_full(samplers):
    for s in samplers.values():
        tab = s._coef_table()
        for index in range(DDIM_STEPS):
            want = torch.cat([c.float().reshape(1) for c in ddim_coefs(s, index, False, "cpu", 1)])
            assert torch.equal(tab[index], want), index
        for index in (0, 1, 499, 999):
            want = torch.cat([c.float().reshape(1) for c in ddim_coefs(s, index, True, "cpu", 1)])
            assert torch.equal(s._coef_original(index)[0], want), index


# ------------------------------------------------------------------------------------------------- GEGLU gate
def _gate_errors(coef):
    g = all_finite_f16()
    out = torch.from_numpy(gelu_sig_model(g.float().numpy(), coef)).half()
    return geglu_gate_errors(out, g), out, g


def test_gelu_sig_model_within_bound():
    err, out, g = _gate_errors(GELU_SIG_COEF)
    gs = torch.from_numpy(gelu_sig_model(g.float().numpy())).double()
    dev = (gs - gelu64(g)).abs()
    inside = g.abs() <= 10
    off = int((bits(out) != bits(gelu64(g).half())).sum())
    print(f"[gelu_sig model] max err/bound {err.max().item():.3f}; fp32 |gelu_sig - gelu| max "
          f"{dev[inside].max().item():.3g} on [-10, 10], {dev[(g >= -10) & (g <= -8)].max().item():.3g} on [-10, -8], "
          f"{dev[~inside].max().item():.3g} beyond; {off} gates differ from fp16(gelu)")
    assert err.max().item() <= 1.0
    assert dev[inside].max().item() < 2.6e-5 and dev[(g.abs() >= 8) & inside].max().item() < 3e-8
    assert (dev[~inside] <= 3e-9 * g[~inside].double().abs()).all()


@pytest.mark.parametrize("which", range(3))
def test_gelu_sig_check_rejects_coefficient_off(which):
    coef = list(GELU_SIG_COEF)
    coef[which] *= 1 + 1e-3
    err, _, _ = _gate_errors(tuple(coef))
    print(f"[gelu_sig mutant] coefficient {which} x (1 + 1e-3): max err/bound {err.max().item():.3f}, "
          f"{int((err > 1).sum())} gates outside")
    assert err.max().item() > 1.0


# ------------------------------------------------------------------------------------------------- Swin windows
@pytest.mark.parametrize("H,W,C", WINDOW_GEOMETRIES)
def test_window_maps_match_reference(H, W, C):
    B = 2
    x = torch.arange(B * H * W, dtype=torch.float64).reshape(B, H, W, 1) + 1    # pixel ids, 0 = pad
    for ws in WINDOW_SIZES:
        for shift in (0, ws // 2):
            win = apply_gather_index(x, window_gather_index(B, H, W, ws, shift), ws)
            assert torch.equal(win, window_gather_ref(x, ws, shift)), (ws, shift)
            back = apply_scatter_index(win, window_scatter_index(B, H, W, ws, shift), B, H, W)
            assert torch.equal(back, window_scatter_ref(win, B, H, W, ws, shift)), (ws, shift)
            assert torch.equal(back, x), (ws, shift)


@pytest.mark.parametrize("H,W", [(128, 128), (13, 29), (16, 16)])
def test_window_checks_reject_mutants(H, W):
    # a grid of one padded window (H, W <= ws, e.g. 8 x 8) cannot tell the shift's sign: there Hp = 2 * shift
    B, ws, shift = 1, 12, 6
    x = torch.arange(B * H * W, dtype=torch.float64).reshape(B, H, W, 1) + 1
    win = apply_gather_index(x, window_gather_index(B, H, W, ws, shift, "no_wrap"), ws)
    assert not torch.equal(win, window_gather_ref(x, ws, shift)), "gather without the wrap is not rejected"
    good = window_gather_ref(x, ws, shift)
    back = apply_scatter_index(good, window_scatter_index(B, H, W, ws, shift, "shift_sign"), B, H, W)
    assert not torch.equal(back, x), "scatter with the shift sign flipped is not rejected"
