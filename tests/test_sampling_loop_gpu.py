"""GPU checks of the sampling loop shared by DDIMSampler and Sampler (pfd_b200/loop.py), in deterministic mode: every
way a loop runs (one whole-loop graph, graphs of fewer steps, one graph per step with host noise in between, eager)
gives the same bits, and a temperature baked into a captured update is part of the graph cache key."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def assert_same(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), \
        f"{what}: not bit-identical (max abs diff {(a.float() - b.float()).abs().max().item():.3g})"


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
    inp["cond2"] = seeded((2, 148, 768), 80, 0.5).cuda().half()
    inp["x0"] = seeded((2, 4, 16, 16), 81).cuda().half()
    return net, inp


@pytest.fixture
def det():
    import pfd_b200
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(True)
    yield
    pfd_b200.set_deterministic(was)


def _sample(net, inp, kind, sampler=None, eta=0.0, img2img=False, temperature=1.0, steps=8, seed=0, seeds=None,
            **opts):
    """One batch-2 request at 16x16 with CFG, torch's generator reset to `seed` first (seeds: per-sample seeds)."""
    from pfd_b200 import DDIMSampler, Sampler
    cond = inp["cond2"]
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": 2.0, "control": None}
    x_info = {"type": "image"} if seeds is None else {"type": "image", "seeds": seeds}
    if img2img:
        x_info.update(x0=inp["x0"], x0_forward_timesteps=5)
    torch.manual_seed(seed)
    if kind == "ddim":
        s = sampler or DDIMSampler(net, **opts)
        x, inter = s.sample(steps=steps, shape=[2, 4, 16, 16], x_info=x_info, c_info=c_info, verbose=False, eta=eta,
                            temperature=temperature, log_every_t=1)
    else:
        s = sampler or Sampler(net, type=kind, **opts)
        x, inter = s.sample(steps=steps, shape=[2, 4, 16, 16], x_info=x_info, c_info=c_info, eta=eta, log_every_t=1)
    return x.clone(), inter


def _assert_runs_equal(a, b, what):
    assert_same(a[0], b[0], f"{what}: final latent")
    for key in ("pred_xt", "pred_x0"):
        assert len(a[1][key]) == len(b[1][key])
        for k, (u, v) in enumerate(zip(a[1][key], b[1][key])):
            assert_same(u, v, f"{what}: {key}[{k}]")


@pytest.mark.parametrize("kind,eta,img2img", [("ddim", 0.5, False), ("ddim", 0.5, True), ("euler_a", 1.0, False),
                                              ("dpmpp_2m_sde", 1.0, False)])
def test_unseeded_stochastic_graph_equals_eager(env, det, kind, eta, img2img):
    """One-step graph replays with host noise in between give the bits of the eager loop drawing the same noise."""
    net, inp = env
    graph = _sample(net, inp, kind, eta=eta, img2img=img2img)
    eager = _sample(net, inp, kind, eta=eta, img2img=img2img, use_cuda_graph=False)
    _assert_runs_equal(graph, eager, f"{kind} eta {eta}{' img2img' if img2img else ''}: graph vs eager")
    other = _sample(net, inp, kind, eta=eta, img2img=img2img, seed=1)
    assert (other[0].float() - graph[0].float()).abs().max().item() > 0.01, "the noise did not reach the update"


def test_ddim_eta0_graph_lengths_are_bit_identical(env, det):
    net, inp = env
    whole = _sample(net, inp, "ddim")
    for opts in ({"steps_per_graph": 4}, {"steps_per_graph": 1}, {"use_cuda_graph": False}):
        _assert_runs_equal(_sample(net, inp, "ddim", **opts), whole, f"DDIM eta 0 {opts} vs one whole-loop graph")


@pytest.mark.parametrize("seeded", [False, True])
def test_ddim_temperature_is_part_of_the_cache_key(env, det, seeded):
    """A sampler that captured eta > 0 at temperature 1.0 must not replay that graph for a request at 0.5."""
    from pfd_b200 import DDIMSampler
    net, inp = env
    smp = DDIMSampler(net)

    def run(sampler, temperature):
        return _sample(net, inp, "ddim", sampler=sampler, eta=0.5, temperature=temperature,
                       seeds=7 if seeded else None)[0]

    t1 = run(smp, 1.0)
    t05 = run(smp, 0.5)
    assert len(smp._states) == 2
    assert_same(t05, run(DDIMSampler(net), 0.5), "temperature 0.5 after 1.0 vs a fresh sampler at 0.5")
    assert (t05.float() - t1.float()).abs().max().item() > 1e-3, "temperature 0.5 gave the temperature 1.0 result"
