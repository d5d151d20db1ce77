"""CPU checks of the k-diffusion samplers (Euler ancestral, DPM-Solver++(2M)): the float64 oracle against the unmodified
reference's schedule and Euler-ancestral loop (tests/golden/sampler_reference.npz, tools/make_golden_sampler.py), the
oracle's convergence order on a Gaussian whose probability-flow ODE has a closed form, and the host-side schedule /
coefficient tables of pfd_b200.sampler against the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import pfd_oracle as PO
from oracle import sampler_oracle as SO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampler_reference.npz")
NS = (1, 10, 20, 25, 50)


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _ac(tag):
    ac = PO.schedule_buffers()["alphas_cumprod"]
    return ac.half() if tag == "fp16" else ac


@pytest.mark.parametrize("tag", ["fp32", "fp16"])
@pytest.mark.parametrize("n", NS)
def test_oracle_schedule_matches_reference(gold, n, tag):
    ref = gold[f"sigmas_{n}_{tag}"]
    got = SO.get_sigmas(_ac(tag), n).numpy()
    assert got.shape == ref.shape == (n + 1,) and got[-1] == 0 == ref[-1]
    np.testing.assert_allclose(got[:-1], ref[:-1], rtol=1e-6, atol=0)


def test_fp16_alphas_cumprod_moves_the_schedule(gold):
    # net.half() rounds alphas_cumprod; the schedule is built from the rounded buffer (App. C #6 of SURVEY.md)
    assert abs(gold["sigmas_20_fp32"][-2] - 0.0292) < 5e-5 and abs(gold["sigmas_20_fp16"][-2] - 0.0313) < 5e-5


def test_oracle_euler_ancestral_table_reproduces_reference_trajectories(gold):
    mu_seed, s = gold["gauss"]
    mu = torch.randn(tuple(gold["shape"]), generator=torch.Generator().manual_seed(int(mu_seed)))
    den = SO.gaussian_denoiser(mu, float(s))
    i = 0
    while f"ea_{i}_case" in gold:
        seed, n, f16 = (int(v) for v in gold[f"ea_{i}_case"])
        sigmas = SO.get_sigmas(_ac("fp16" if f16 else "fp32"), n)
        np.testing.assert_allclose(sigmas.numpy(), gold[f"ea_{i}_sigmas"], rtol=1e-6)
        sigmas = torch.as_tensor(gold[f"ea_{i}_sigmas"])          # the reference's own fp32 values from here on
        torch.manual_seed(seed)
        xt = torch.randn(tuple(gold["shape"]))
        assert torch.equal(xt, torch.as_tensor(gold[f"ea_{i}_xt"]))
        noises = [torch.randn_like(xt) if sigmas[k + 1] > 0 else None for k in range(n)]
        trace = []
        out = SO.run_table(den, xt * sigmas[0], SO.coef_table("euler_a", sigmas, 1.0), noises, trace)
        xs = gold[f"ea_{i}_xs"]
        assert len(trace) == len(xs) == n
        for k, (x, _) in enumerate(trace):
            ref = torch.as_tensor(xs[k]).double()
            err = (x - ref).abs().max().item() / ref.abs().max().item()
            assert err < 2e-6, (i, k, err)
        ref = torch.as_tensor(gold[f"ea_{i}_out"]).double()
        assert (out - ref).abs().max().item() / ref.abs().max().item() < 2e-6
        # the plain k-diffusion loop and the coefficient table are the same computation
        kd = SO.sample_euler_ancestral(den, xt * sigmas[0], sigmas, 1.0, noises)
        assert (kd - out).abs().max().item() < 1e-12
        i += 1
    assert i >= 2


def _ode_error(kind, n, eta=0.0):
    mu = torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(3)).double()
    s = 0.5
    # log-uniform steps over the model's sigma range, ending at sigma_min (not 0): the uniform-in-t grid of get_sigmas
    # has a last step whose log-sigma length shrinks only like log(1 + 1000/n), which hides the asymptotic order
    sigmas = torch.logspace(np.log10(14.6), np.log10(0.03), n + 1, dtype=torch.float64)
    xT = torch.randn((2, 4, 8, 8), generator=torch.Generator().manual_seed(4)).double() * float(sigmas[0])
    den = SO.gaussian_denoiser(mu, s)
    x = SO.run_table(den, xT, SO.coef_table(kind, sigmas, eta))
    exact = SO.gaussian_ode_solution(mu, s, xT, float(sigmas[0]), float(sigmas[-1]))
    if kind == "dpmpp_2m":
        assert (SO.sample_dpmpp_2m(den, xT, sigmas) - x).abs().max().item() < 1e-12
    return (x - exact).pow(2).mean().sqrt().item()


@pytest.mark.parametrize("kind,order", [("euler_a", 1), ("dpmpp_2m", 2)])
def test_convergence_order_on_gaussian_ode(kind, order):
    errs = [_ode_error(kind, n) for n in (20, 40, 80, 160)]
    ratios = [errs[k] / errs[k + 1] for k in range(len(errs) - 1)]
    expect = 2.0 ** order
    print(kind, errs, ratios)
    assert all(0.75 * expect < r < 1.35 * expect for r in ratios[1:]), (kind, errs, ratios)


def test_sigma_to_t_inverts_the_schedule():
    for tag in ("fp32", "fp16"):
        ac = _ac(tag)
        ls = SO.log_sigmas(ac)
        t = torch.linspace(999, 0, 25).double()
        sig = SO.get_sigmas(ac, 25)[:-1]
        assert (SO.sigma_to_t(sig, ls) - t).abs().max().item() < 1e-6
        ti = torch.tensor([999.0, 801.0, 1.0, 0.0], dtype=torch.float64)
        assert torch.equal(SO.sigma_to_t(ls[ti.long()].exp(), ls), ti)


# ----------------------------------------------------------------------------- product host code (no GPU calls)
@pytest.mark.parametrize("tag", ["fp32", "fp16"])
def test_product_schedule_and_timesteps_match_oracle(tag):
    from pfd_b200 import sampler as S
    ac = _ac(tag)
    for n in NS:
        np.testing.assert_allclose(S.get_sigmas(ac, n).double().numpy(), SO.get_sigmas(ac, n).numpy(), rtol=1e-6)
        np.testing.assert_array_equal(S.schedule_timesteps(n, 1000), torch.linspace(999, 0, n).double().numpy())
    sig = np.array([14.6, 7.3, 2.0, 0.5, 0.1, 0.03], dtype=np.float64)
    np.testing.assert_allclose(S.sigma_to_t(sig, S.model_log_sigmas(ac)),
                               SO.sigma_to_t(torch.as_tensor(sig), SO.log_sigmas(ac)).numpy(), rtol=0, atol=1e-9)


@pytest.mark.parametrize("kind,eta", [("euler_a", 1.0), ("euler_a", 0.0), ("euler_a", 0.5), ("dpmpp_2m", 0.0)])
def test_product_coefficient_tables_match_oracle(kind, eta):
    from pfd_b200 import sampler as S
    for sig in (SO.get_sigmas(_ac("fp16"), 20).numpy(), SO.get_sigmas(_ac("fp32"), 7).numpy()[:-1]):
        np.testing.assert_allclose(S.coef_table(kind, sig, eta), SO.coef_table(kind, sig, eta).numpy(),
                                   rtol=1e-12, atol=1e-12)


def test_log_steps_follow_the_ddim_rule():
    from pfd_b200 import sampler as S
    assert S.log_steps(8, 100) == [0, 7]
    assert S.log_steps(50, 10) == [0, 9, 19, 29, 39, 49]
    assert S.log_steps(1, 100) == [0]


def test_sampler_rejects_unknown_types_and_img2img():
    from pfd_b200 import Sampler
    with pytest.raises(ValueError):
        Sampler(object(), type="heun")

    class Net:
        alphas_cumprod = PO.schedule_buffers()["alphas_cumprod"]
    with pytest.raises(NotImplementedError):
        Sampler(Net(), type="eular_a").sample(steps=4, shape=[1, 4, 8, 8], x_info={"type": "image", "x0": 1},
                                              c_info={})
