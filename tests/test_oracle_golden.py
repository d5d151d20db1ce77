"""CPU tests: the oracle (oracle/pfd_oracle.py) reproduces the golden outputs that tools/make_golden.py
recorded from the UNMODIFIED reference (fp32, CPU, name-seeded synthetic weights), the product's
module tree exposes exactly the reference's state-dict keys/shapes, and the host-side schedule
logic matches the closed forms."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import pfd_oracle as O
from oracle.golden_inputs import golden_inputs
from pfd_b200.weights import SCHEDULE_BUFFERS, synth_state_dict

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def shapes():
    return json.load(open(os.path.join(GOLD, "state_dict_shapes.json")))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLD, "reference_outputs.npz")))


def _sd(shapes, prefix):
    return O.sub(synth_state_dict(shapes, seed=0, prefix=prefix), prefix)


def _close(out, ref, tol=2e-4):
    ref = torch.as_tensor(ref).float()
    d = (out.float() - ref).abs().max().item()
    assert d <= tol * max(1.0, ref.abs().max().item()), f"max dev {d}"


def test_pin_report_says_oracle_matches_reference():
    rep = json.load(open(os.path.join(GOLD, "oracle_pin_report.json")))
    assert max(rep["max_abs_dev_reference_vs_oracle"].values()) < 1e-4


def test_product_state_dict_matches_reference_layout(shapes):
    from pfd_b200 import get_model, model_cfg_bank
    with torch.device("meta"):
        net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet"))
    sd = net.state_dict()
    assert set(sd) == set(shapes)
    for k, v in sd.items():
        assert list(v.shape) == shapes[k][0], k
        assert str(v.dtype).replace("torch.", "") == shapes[k][1], k


def test_schedule_buffers_and_ddim_timesteps():
    buf = O.schedule_buffers()
    assert abs(buf["betas"][0].item() - 0.00085) < 1e-9 and abs(buf["betas"][-1].item() - 0.012) < 1e-8
    assert torch.allclose(buf["alphas_cumprod"], torch.cumprod(1 - buf["betas"].double(), 0).float(), atol=1e-6)
    assert len(O.ddim_timesteps(10)) == 10 and len(O.ddim_timesteps(50)) == 50 and len(O.ddim_timesteps(30)) == 31
    assert O.ddim_timesteps(50)[0] == 1 and O.ddim_timesteps(50)[-1] == 981
    # the product's host-side schedule is the same arithmetic
    from pfd_b200 import get_model, model_cfg_bank
    from pfd_b200.ddim import DDIMSampler, make_ddim_timesteps
    assert list(make_ddim_timesteps(30, 1000)) == list(O.ddim_timesteps(30))

    class Stub:
        num_timesteps = 1000
        betas, alphas_cumprod, alphas_cumprod_prev = buf["betas"], buf["alphas_cumprod"], buf["alphas_cumprod_prev"]
    s = DDIMSampler(Stub())
    s.make_schedule(50, ddim_eta=0.0)
    ts, a, ap, sg, s1m = O.ddim_schedule(buf["alphas_cumprod"], 50, 0.0)
    assert np.array_equal(s.ddim_timesteps, ts) and torch.equal(s.ddim_alphas, a)
    assert np.array_equal(s.ddim_alphas_prev, ap) and np.allclose(np.asarray(s.ddim_sqrt_one_minus_alphas), np.asarray(s1m))
    # per-step coefficient table fed to pfd_ddim_step_f16: the fp16 roundings torch.full(..., dtype=float16) applies
    tab = s._coef_table("cpu")
    assert tab.shape == (50, 4) and tab.dtype == torch.float32
    for i in (0, 17, 49):
        want = [float(a[i].half()), float(torch.tensor(ap[i]).half()), 0.0, float(torch.as_tensor(s1m[i]).half())]
        assert tab[i].tolist() == want
    # eta > 0: sigma_t of ddim.py:44-48 lands in column 2; the img2img branch walks a prefix of the same table
    s.make_schedule(50, ddim_eta=0.5)
    _, a2, ap2, sg2, _ = O.ddim_schedule(buf["alphas_cumprod"], 50, 0.5)
    assert np.allclose(np.asarray(s.ddim_sigmas), np.asarray(sg2)) and float(s._coef_table("cpu")[10, 2]) > 0.0


def test_timestep_embedding_formula():
    e = O.timestep_embedding(torch.tensor([0, 1, 981]), 320)
    assert e.shape == (3, 320) and torch.allclose(e[0, :160], torch.ones(160)) and torch.allclose(e[0, 160:], torch.zeros(160))
    assert abs(e[1, 160].item() - np.sin(1.0)) < 1e-6


def test_unet_and_controlnet_match_reference_golden(shapes, gold):
    inp = golden_inputs()
    usd = _sd(shapes, "diffuser.image.")
    with torch.no_grad():
        eps = O.unet_apply(usd, O.UNET_SD15, inp["x"], inp["t"], inp["ctx"])
        _close(eps, gold["unet_eps"])
        csd = _sd(shapes, "ctl.")
        outs = O.controlnet_apply(csd, O.CONTROLNET_SD15, inp["x"], inp["hint"], inp["t"], inp["ctx"])
        for i, o in enumerate(outs):
            _close(o.reshape(-1)[::37], gold[f"ctl_{i}_sub"])
        eps = O.unet_apply(usd, O.UNET_SD15, inp["x"], inp["t"], inp["ctx"], control=outs)
        _close(eps, gold["unet_eps_control"])
        buf = O.schedule_buffers()
        x = O.ddim_sample(usd, O.UNET_SD15, buf["alphas_cumprod"], steps=4, x_T=inp["x_T"], cond=inp["cond"],
                          uncond=torch.zeros_like(inp["cond"]), guidance=2.0)
        _close(x, gold["ddim4_latent"])


def test_vae_decode_matches_reference_golden(shapes, gold):
    with torch.no_grad():
        im = O.vae_decode(_sd(shapes, "vae.image."), O.VAE_SD, golden_inputs()["z"])
    _close(im, gold["vae_image"])


def test_seecoder_matches_reference_golden(shapes, gold):
    inp = golden_inputs()
    ssd = _sd(shapes, "ctx.image.")
    with torch.no_grad():
        fea = O.swin_forward(O.sub(ssd, "imencoder."), O.SWIN_L, inp["img"])
        for k in ("res3", "res4", "res5"):
            _close(fea[k].reshape(-1)[::11], gold[f"swin_{k}_sub"])
        c = O.seecoder_encode(ssd, inp["img"])
    _close(c, gold["seecoder_ctx"].astype(np.float32), tol=2e-3)          # golden stored as fp16


def test_ddim_update_edge_cases():
    x = torch.randn(2, 4, 8, 8)
    e = torch.zeros_like(x)
    xp, p0 = O.ddim_update(x, e, 0.5, 0.7, 0.0, np.sqrt(0.5))
    assert torch.allclose(p0, x / np.sqrt(0.5), atol=1e-6) and torch.allclose(xp, np.sqrt(0.7) * p0, atol=1e-6)
    # a_t == a_prev and eps consistent with x = sqrt(a) x0 + sqrt(1-a) eps  ->  x_prev == x (idempotence)
    x0, eps = torch.randn(2, 4, 8, 8), torch.randn(2, 4, 8, 8)
    a = 0.6
    xt = np.sqrt(a) * x0 + np.sqrt(1 - a) * eps
    xp, p0 = O.ddim_update(xt, eps, a, a, 0.0, np.sqrt(1 - a))
    assert torch.allclose(p0, x0, atol=1e-5) and torch.allclose(xp, xt, atol=1e-5)


def test_swin_mask_and_index_builders_agree_with_product():
    from pfd_b200.swin import relative_position_index, shift_mask
    assert torch.equal(relative_position_index(12), O.relative_position_index(12))
    for (H, W) in [(32, 32), (16, 20), (8, 8)]:
        assert torch.equal(shift_mask(H, W, 12, 6), O.swin_shift_mask(H, W, 12, 6, torch.float32))


# ---- round 2: the oracle's eta / VAE-encode / multicontext restatements against the reference's outputs at the
#      config fixtures (tests/golden/config_outputs.npz, tools/make_golden_configs.py); the cheap cases run here,
#      the full-size ones (64x64 / 96x96 latents) are compared with the CUDA path in tests/test_configs_gpu.py.
@pytest.fixture(scope="module")
def cgold():
    return dict(np.load(os.path.join(GOLD, "config_outputs.npz")))


def test_oracle_eta_sampler_matches_reference(shapes, cgold):
    from oracle.golden_inputs import config_inputs
    inp = config_inputs()
    usd = _sd(shapes, "diffuser.image.")
    with torch.no_grad():
        x = O.ddim_sample(usd, O.UNET_SD15, O.schedule_buffers()["alphas_cumprod"], steps=4, x_T=inp["c7_xT"],
                          cond=inp["c7_cond"], uncond=torch.zeros_like(inp["c7_cond"]), guidance=2.0, eta=0.5,
                          noises=inp["c7_noise"])
    _close(x, cgold["c7_latent"])


def test_oracle_vae_encode_matches_reference(shapes, cgold):
    from oracle.golden_inputs import config_inputs
    inp = config_inputs()
    with torch.no_grad():
        mean, logvar = O.vae_encode_moments(_sd(shapes, "vae.image."), O.VAE_SD, inp["c8_img"])
    _close(mean, cgold["c8_mean"])
    _close(logvar, cgold["c8_logvar"])
    nz = torch.randn(mean.shape, generator=torch.Generator().manual_seed(0))
    z = O.vae_encode(_sd(shapes, "vae.image."), O.VAE_SD, inp["c8_img"], nz)
    assert torch.allclose(z, 0.18215 * (mean + torch.exp(0.5 * logvar) * nz), atol=1e-6)


def test_oracle_multicontext_matches_reference(shapes, cgold):
    from oracle.golden_inputs import config_inputs
    inp = config_inputs()
    usd = _sd(shapes, "diffuser.image.")
    ca, cb = inp["c9_cond_a"], inp["c9_cond_b"]
    with torch.no_grad():
        x = O.ddim_sample(usd, O.UNET_SD15, O.schedule_buffers()["alphas_cumprod"], steps=4, x_T=inp["c9_xT"],
                          cond=None, uncond=None, guidance=2.0,
                          mixed=[(ca, torch.zeros_like(ca), 0.3), (cb, torch.zeros_like(cb), 0.7)])
    _close(x, cgold["c9_latent"])


def test_config_fixture_is_complete(cgold):
    need = ["c1_ctx", "c1_latent", "c1_image", "c2_eps_t981", "c2_eps_t501", "c2_eps_t1", "c3_eps", "c4_eps",
            "c5_ctx", "c5_x_step0", "c5_x_step1", "c6_ctx", "c7_latent", "c8_mean", "c8_logvar", "c9_latent"]
    assert all(k in cgold for k in need), [k for k in need if k not in cgold]
    assert tuple(cgold["c2_eps_t501__shape"]) == (8, 4, 64, 64) and tuple(cgold["c5_x_step1__shape"]) == (1, 4, 96, 96)
    assert tuple(cgold["c1_image__shape"]) == (1, 3, 512, 512) and cgold["c5_x_step0"].shape == (1, 4, 96, 96)
