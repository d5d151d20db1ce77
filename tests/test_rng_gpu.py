"""GPU checks of per-sample seeds (x_info["seeds"], pfd_b200.randn, pfd_randn_f16): the kernel against the numpy
transcription of the generator, batch invariance of every seeded sampler in deterministic mode, the whole-loop graphs
(replay equals the eager run, one capture serves every seed), and the seeded stochastic samplers (euler_a,
dpmpp_2m_sde) against the float64 oracle loop fed the same noise."""
import math

import numpy as np
import pytest
import torch

from tools.rng_reference import randn_batch64

pytestmark = pytest.mark.gpu


def _assert_fp16_of(got, ref64):
    """got (fp16) is ref64 rounded to fp16: within one fp16 ulp of the float64 value."""
    g, r = got.double().cpu(), torch.as_tensor(ref64).double()
    ulp = torch.clamp(r.abs(), min=2.0 ** -14) * 2.0 ** -10
    err = ((g - r).abs() / ulp).max().item()
    assert err <= 1.0, err


def assert_same(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), \
        f"{what}: not bit-identical (max abs diff {(a.float() - b.float()).abs().max().item():.3g})"


# ----------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("B,n", [(1, 1024), (7, 1023), (3, 6), (2, 1), (4, 4 * 64 * 64)])
def test_kernel_matches_reference(B, n):
    from pfd_b200 import native as nv
    from pfd_b200.rng import seeds_tensor
    seeds = np.array([17 + 1000 * b for b in range(B)], dtype=np.uint64)
    seeds[-1] = np.uint64(2 ** 64 - 5)                           # both key words in use
    sd = seeds_tensor(seeds, "cuda")
    for stream, draw, scale in ((0, 0, 1.0), (1, 9, 1.0), (2, 0, 0.37)):
        out = torch.full((B, n), 7.0, dtype=torch.float16, device="cuda")
        nv.randn_f16(out, sd, stream, draw, scale=scale)
        _assert_fp16_of(out, randn_batch64(seeds, n, stream, draw, scale))
    # the draw index taken from a device counter: draw + *draw_dev
    out = torch.empty((B, n), dtype=torch.float16, device="cuda")
    nv.randn_f16(out, sd, 1, 2, torch.tensor([5], dtype=torch.int32, device="cuda"))
    _assert_fp16_of(out, randn_batch64(seeds, n, 1, 7))


def test_public_randn():
    import pfd_b200
    x = pfd_b200.randn((3, 4, 5, 5), 40, stream=1, draw=2)
    assert x.dtype == torch.float16 and x.shape == (3, 4, 5, 5) and x.is_cuda
    _assert_fp16_of(x.reshape(3, -1), randn_batch64([40, 41, 42], 100, 1, 2))
    assert_same(pfd_b200.randn((1, 4, 5, 5), [41], stream=1, draw=2)[0], x[1], "seed 41 alone vs in a batch")
    assert_same(pfd_b200.randn((2, 4, 5, 5), torch.tensor([42, 40]), 1, 2), x[[2, 0]], "tensor seeds")
    with pytest.raises(ValueError):
        pfd_b200.randn((2, 4), [1, 2, 3])


# ----------------------------------------------------------------------------------------------- samplers
@pytest.fixture(scope="module")
def env():
    from oracle.golden_inputs import golden_inputs, seeded
    from pfd_b200 import get_model, model_cfg_bank
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    net.eval()
    inp = {k: v.cuda() for k, v in golden_inputs().items()}
    # per-seed inputs: a seed always comes with the same conditioning and (img2img) x0, wherever it sits in the batch
    inp["bank"] = {s: (seeded((1, 148, 768), 80 + i, 0.5).cuda().half(), seeded((1, 4, 16, 16), 90 + i).cuda().half())
                   for i, s in enumerate((101, 202, 303, 404, 505, 2 ** 63 + 7))}
    return net, inp


@pytest.fixture
def det():
    import pfd_b200
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(True)
    yield
    pfd_b200.set_deterministic(was)


CASES = {  # name -> (sampler type, eta, img2img)
    "ddim_eta0.5": ("ddim", 0.5, False),
    "ddim_img2img": ("ddim", 0.5, True),
    "euler_a": ("euler_a", 1.0, False),
    "dpmpp_2m_sde": ("dpmpp_2m_sde", 1.0, False),
}


def _sample(net, inp, case, seeds, sampler=None, graph=True, control=False, steps=4):
    from pfd_b200 import DDIMSampler, Sampler
    kind, eta, img2img = CASES[case]
    cond = torch.cat([inp["bank"][s][0] for s in seeds])
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": 2.0, "control": inp["hint"].half() if control else None}
    shape = [len(seeds), 4, 16, 16]
    x_info = {"type": "image", "seeds": list(seeds)}
    if kind == "ddim":
        if img2img:
            x_info.update(x0=torch.cat([inp["bank"][s][1] for s in seeds]), x0_forward_timesteps=3)
        s = sampler or DDIMSampler(net, use_cuda_graph=graph)
        x, inter = s.sample(steps=steps, shape=shape, x_info=x_info, c_info=c_info, verbose=False, eta=eta,
                            log_every_t=1)
    else:
        s = sampler or Sampler(net, type=kind, use_cuda_graph=graph)
        x, inter = s.sample(steps=steps, shape=shape, x_info=x_info, c_info=c_info, eta=eta, log_every_t=1)
    return x.clone(), inter


@pytest.mark.parametrize("case", list(CASES))
def test_seeded_samplers_batch_invariant(env, det, case):
    net, inp = env
    s0, s1, s2 = 101, 202, 2 ** 63 + 7
    x3, inter3 = _sample(net, inp, case, [s0, s1, s2])
    x1, inter1 = _sample(net, inp, case, [s1])
    assert_same(x1[0], x3[1], f"{case}: seed {s1} alone vs at position 1 of 3")
    for key in ("pred_xt", "pred_x0"):
        for k, (a, b) in enumerate(zip(inter1[key], inter3[key])):
            assert_same(a[0], b[1], f"{case} {key}[{k}]")
    x5, _ = _sample(net, inp, case, [303, 404, 505, s1, s0])
    assert_same(x5[3], x3[1], f"{case}: seed {s1} at position 3 of 5 vs position 1 of 3")
    assert_same(x5[4], x3[0], f"{case}: seed {s0} at position 4 of 5 vs position 0 of 3")
    assert (x3[0].float() - x3[1].float()).abs().max().item() > 0.1


@pytest.mark.parametrize("case", list(CASES))
def test_seeded_graph_matches_eager_and_serves_every_seed(env, det, case):
    from pfd_b200 import DDIMSampler, Sampler
    net, inp = env
    kind = CASES[case][0]
    smp = DDIMSampler(net) if kind == "ddim" else Sampler(net, type=kind)
    a, _ = _sample(net, inp, case, [101, 202], sampler=smp)
    assert len(smp._states) == 1
    st = next(iter(smp._states.values()))
    assert st.step_graph is not None and st.prep_graph is not None
    eager, _ = _sample(net, inp, case, [101, 202], graph=False)
    assert_same(a, eager, f"{case}: graph replay vs eager")
    # other seeds (same conditioning) go through the same captured graph and change the output
    cond_bank = inp["bank"]
    saved = dict(cond_bank)
    cond_bank[303], cond_bank[404] = cond_bank[101], cond_bank[202]
    try:
        b, _ = _sample(net, inp, case, [303, 404], sampler=smp)
    finally:
        cond_bank.clear()
        cond_bank.update(saved)
    assert len(smp._states) == 1 and next(iter(smp._states.values())) is st
    assert (a.float() - b.float()).abs().max().item() > 0.1
    assert_same(_sample(net, inp, case, [101, 202], sampler=smp)[0], a, f"{case}: replay after other seeds")


def test_unseeded_requests_keep_their_graphs(env):
    """A seeded request and an unseeded one of the same shape are different captures."""
    from pfd_b200 import Sampler
    net, inp = env
    smp = Sampler(net, type="euler_a")
    cond = inp["bank"][101][0]
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": 2.0, "control": None}
    torch.manual_seed(3)
    smp.sample(steps=4, shape=[1, 4, 16, 16], x_info={"type": "image"}, c_info=dict(c_info), eta=1.0)
    smp.sample(steps=4, shape=[1, 4, 16, 16], x_info={"type": "image", "seeds": 5}, c_info=dict(c_info), eta=1.0)
    assert len(smp._states) == 2
    with pytest.raises(ValueError):
        smp.sample(steps=4, shape=[1, 4, 16, 16], x_info={"type": "image", "seeds": [1, 2]}, c_info=dict(c_info))


# ----------------------------------------------------------------------------------------------- accuracy
def _rel(out, ref):
    out, ref = out.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    return ((out - ref).pow(2).mean() / ref.pow(2).mean()).sqrt().item()


def _oracle_denoiser(net, inp, control, guidance=2.0):
    """D(x, sigma) = x - sigma * CFG(eps), eps from the torch oracle of the UNet (+ ControlNet) in fp16 on the GPU at the
    fp16 UNet input x*c_in and the float timestep t(sigma)."""
    from oracle import pfd_oracle as PO
    from pfd_b200 import sampler as S
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    usd, csd = PO.sub(sd, "diffuser.image."), PO.sub(sd, "ctl.")
    ls = S.model_log_sigmas(net.alphas_cumprod)
    cond = inp["cond"].half()
    c_in = torch.cat([torch.zeros_like(cond), cond])
    hint = inp["hint"].half()

    def denoise(x, sigma):
        cin = 1.0 / math.sqrt(sigma * sigma + 1.0)
        xin = (x * cin).half()
        t = float(S.sigma_to_t([sigma], ls)[0])
        xx = torch.cat([xin, xin])
        tt = torch.full((2,), t, dtype=torch.float32, device=xin.device)
        ctl = PO.controlnet_apply(csd, PO.CONTROLNET_SD15, xx, hint, tt, c_in) if control else None
        eu, ec = PO.unet_apply(usd, PO.UNET_SD15, xx, tt, c_in, ctl).double().chunk(2)
        return x.double() - sigma * (eu + guidance * (ec - eu))
    return denoise


@pytest.mark.parametrize("kind,control", [("euler_a", False), ("dpmpp_2m_sde", False), ("dpmpp_2m_sde", True)])
def test_seeded_sampler_matches_oracle_loop(env, kind, control):
    import pfd_b200
    from oracle import sampler_oracle as SO
    from pfd_b200 import Sampler
    from pfd_b200 import sampler as S
    net, inp = env
    steps, seed, shape = 8, 77, (1, 4, 16, 16)
    cond = inp["cond"].half()
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": 2.0, "control": inp["hint"].half() if control else None}
    x, _ = Sampler(net, type=kind).sample(steps=steps, shape=list(shape), x_info={"type": "image", "seeds": seed},
                                          c_info=c_info, eta=1.0)
    sig = Sampler(net).get_sigmas(steps).double().numpy()
    xt = pfd_b200.randn(shape, seed, stream=0)
    noises = [pfd_b200.randn(shape, seed, stream=1, draw=k) for k in range(steps)]
    # euler_a: the oracle's own table; dpmpp_2m_sde: the product table, which tests/test_rng_cpu.py pins to k-diffusion
    tab = SO.coef_table(kind, sig, 1.0) if kind == "euler_a" else torch.as_tensor(S.coef_table(kind, sig, 1.0))
    with torch.no_grad():
        ref = SO.run_table(_oracle_denoiser(net, inp, control), xt.double() * float(sig[0]), tab, noises)
    rel = _rel(x, ref)
    print(f"[rng] seeded {kind} ({'control' if control else 'plain'}) final latent vs float64 oracle: rel_rms={rel:.3e}")
    assert np.isfinite(rel) and rel <= 1.5e-3, rel
