"""CPU checks of per-sample seeds: the numpy Philox4x32-10 transcription against the published known-answer vectors,
the statistics of the Box-Muller output, seed parsing and the multi-GPU seed split, and the DPM-Solver++(2M) SDE
coefficient table against a float64 transcription of k-diffusion's loop."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import pfd_oracle as PO
from oracle import sampler_oracle as SO
from tools.rng_reference import philox4x32_10, randn64


# ----------------------------------------------------------------------------------------------- generator
@pytest.mark.parametrize("ctr,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, expect):
    got = tuple(int(w) for w in philox4x32_10(ctr, key))
    assert got == expect, [hex(w) for w in got]


N_STAT = 1 << 20


@pytest.fixture(scope="module")
def draws():
    """1M draws each of: seeds s0, s0+1 (stream 0, draw 0), stream 1 and draw 1 of s0, and a seed above 2^32."""
    s0 = 12345
    return {"a": randn64(s0, N_STAT, 0, 0), "seed+1": randn64(s0 + 1, N_STAT, 0, 0),
            "stream1": randn64(s0, N_STAT, 1, 0), "draw1": randn64(s0, N_STAT, 0, 1),
            "big": randn64((7 << 40) + 3, N_STAT, 2, 5)}


def test_box_muller_statistics(draws):
    z = np.concatenate(list(draws.values()))
    n = z.size
    assert n >= 4 * 10 ** 6
    assert abs(z.mean()) < 5 / math.sqrt(n), z.mean()
    assert abs(z.var() - 1.0) < 5 * math.sqrt(2.0 / n), z.var()
    p = stats.kstest(z, "norm").pvalue
    assert p > 1e-3, p
    for k, v in draws.items():
        assert stats.kstest(v, "norm").pvalue > 1e-3, k
    assert np.all(np.isfinite(z)) and np.abs(z).max() < 7.0


def test_no_correlation_between_seeds_streams_draws_and_elements(draws):
    a = draws["a"]
    pairs = {"adjacent seeds": draws["seed+1"], "streams 0 / 1": draws["stream1"], "draws 0 / 1": draws["draw1"]}
    for what, b in pairs.items():
        r = np.corrcoef(a, b)[0, 1]
        assert abs(r) < 5e-3, (what, r)
    for lag in (1, 2, 3, 4):                 # within a Philox group (lags 1-3) and across groups
        r = np.corrcoef(a[:-lag], a[lag:])[0, 1]
        assert abs(r) < 5e-3, (lag, r)


def test_element_index_is_independent_of_the_range_drawn():
    full = randn64(99, 1001, 1, 3)
    assert np.array_equal(randn64(99, 1001 - 400, 1, 3, first=400), full[400:])
    assert np.array_equal(randn64(99, 7, 1, 3), full[:7])


# ----------------------------------------------------------------------------------------------- seeds
def test_parse_seeds():
    from pfd_b200.rng import parse_seeds
    assert parse_seeds(5, 3).tolist() == [5, 6, 7]
    assert parse_seeds([3, 1, 2], 3).tolist() == [3, 1, 2]
    assert parse_seeds(torch.tensor([9, 0], dtype=torch.int64), 2).tolist() == [9, 0]
    assert parse_seeds([2 ** 64 - 1], 1).tolist() == [2 ** 64 - 1]
    assert parse_seeds(np.array([4, 5], dtype=np.uint64), 2).tolist() == [4, 5]
    for bad, b in (([1, 2], 3), (-1, 1), ([2 ** 64], 1), (2 ** 64 - 1, 2), ([1.5], 1), (True, 1), ("7", 1),
                   (torch.tensor([-3]), 1), (torch.tensor([1.0]), 1), (torch.tensor([1, 2]), 1)):
        with pytest.raises(ValueError):
            parse_seeds(bad, b)


def test_seeds_tensor_keeps_the_bits():
    from pfd_b200.rng import seeds_tensor
    s = np.array([0, 1, 2 ** 63, 2 ** 64 - 1], dtype=np.uint64)
    t = seeds_tensor(s, "cpu")
    assert t.dtype == torch.int64 and t.numpy().view(np.uint64).tolist() == s.tolist()


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_shard_seeds_partition(world):
    from pfd_b200.parallel import shard_range, shard_seeds
    for total in (1, 2, 5, 7, 16):
        seeds = [1000 + 7 * i for i in range(total)]
        parts = [shard_seeds(seeds, world, r) for r in range(world)]
        assert sum(parts, []) == seeds
        for r in range(world):
            a, b = shard_range(total, world, r)
            assert parts[r] == seeds[a:b]
        assert sum((shard_seeds(torch.tensor(seeds), world, r) for r in range(world)), []) == seeds


# ----------------------------------------------------------------------------------------------- DPM++ 2M SDE
def kdiffusion_dpmpp_2m_sde(denoise, x, sigmas, eta, noises):
    """k-diffusion sample_dpmpp_2m_sde (solver_type 'midpoint', s_noise 1, Gaussian noises[i]) in float64."""
    x = x.double()
    s = [float(v) for v in sigmas]
    old, h_last = None, None
    for i in range(len(s) - 1):
        d = denoise(x, s[i]).double()
        if s[i + 1] == 0:
            x = d
        else:
            t, t_next = -math.log(s[i]), -math.log(s[i + 1])
            h = t_next - t
            eta_h = eta * h
            x = s[i + 1] / s[i] * math.exp(-eta_h) * x + (-math.expm1(-h - eta_h)) * d
            if old is not None:
                r = h_last / h
                x = x + 0.5 * (-math.expm1(-h - eta_h)) * (1 / r) * (d - old)
            if eta:
                x = x + noises[i].double() * s[i + 1] * math.sqrt(-math.expm1(-2 * eta_h))
            h_last = h
        old = d
    return x


def _gauss():
    mu = torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(3)).double()
    return mu, 0.5, SO.gaussian_denoiser(mu, 0.5)


@pytest.mark.parametrize("eta", [1.0, 0.5, 0.0])
def test_dpmpp_2m_sde_table_matches_kdiffusion_loop(eta):
    from pfd_b200 import sampler as S
    _, _, den = _gauss()
    for sig in (SO.get_sigmas(PO.schedule_buffers()["alphas_cumprod"].half(), 12).numpy(),
                np.geomspace(14.6, 0.03, 9)):
        g = torch.Generator().manual_seed(11)
        x = torch.randn((2, 4, 8, 8), generator=g).double() * float(sig[0])
        noises = [torch.randn((2, 4, 8, 8), generator=g).double() for _ in range(len(sig) - 1)]
        tab = torch.as_tensor(S.coef_table("dpmpp_2m_sde", sig, eta))
        got = SO.run_table(den, x, tab, noises)
        ref = kdiffusion_dpmpp_2m_sde(den, x, sig, eta, noises)
        assert (got - ref).abs().max().item() < 1e-12 * (ref.abs().max().item() + 1.0)
        # last row of a schedule ending at 0: x' = D, no noise
        if sig[-1] == 0:
            assert tab[-1, 1:5].tolist() == [0.0, 1.0, 0.0, 0.0]


def test_dpmpp_2m_sde_at_eta_0_is_dpmpp_2m():
    from pfd_b200 import sampler as S
    for sig in (SO.get_sigmas(PO.schedule_buffers()["alphas_cumprod"].half(), 20).numpy(), np.geomspace(14.6, 0.03, 9)):
        sde, ode = S.coef_table("dpmpp_2m_sde", sig, 0.0), S.coef_table("dpmpp_2m", sig, 0.0)
        np.testing.assert_allclose(sde, ode, rtol=0, atol=1e-12)
        assert np.all(sde[:, 4] == 0.0)


def test_dpmpp_2m_sde_eta_0_second_order_on_gaussian_ode():
    from pfd_b200 import sampler as S
    mu, s, den = _gauss()
    errs = []
    for n in (20, 40, 80, 160):
        sigmas = torch.logspace(np.log10(14.6), np.log10(0.03), n + 1, dtype=torch.float64)
        xT = torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(4)).double() * float(sigmas[0])
        x = SO.run_table(den, xT, torch.as_tensor(S.coef_table("dpmpp_2m_sde", sigmas.numpy(), 0.0)))
        exact = SO.gaussian_ode_solution(mu, s, xT, float(sigmas[0]), float(sigmas[-1]))
        errs.append((x - exact).pow(2).mean().sqrt().item())
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    assert all(0.75 * 4 < r < 1.35 * 4 for r in ratios[1:]), (errs, ratios)


def test_sampler_types():
    from pfd_b200 import Sampler
    from pfd_b200 import sampler as S
    assert S.TYPES["dpmpp_2m_sde"] == "dpmpp_2m_sde"
    with pytest.raises(ValueError):
        Sampler(object(), type="heun")
    assert Sampler(object(), type="dpmpp_2m_sde").type == "dpmpp_2m_sde"
