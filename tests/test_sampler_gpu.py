"""GPU checks of the k-diffusion samplers (pfd_b200.Sampler: Euler ancestral, DPM-Solver++(2M)): the update kernel and
the float-timestep embedding against float64 restatements, the whole sampler against the float64 oracle loop driving
the torch UNet / ControlNet oracle in fp16, the equivalence of plain Euler on DDIM's timesteps with DDIM, and the
CUDA-graph paths (whole loop, per-step with noise, weight hot swap)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(out, ref):
    out, ref = out.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    mse = (out - ref).pow(2).mean().item()
    return mse, (mse / max(ref.pow(2).mean().item(), 1e-30)) ** 0.5


def _check(name, out, ref, rel_tol, mse_tol=1e-3):
    mse, rel = _rel(out, ref)
    print(f"[sampler] {name}: mse={mse:.3e} rel_rms={rel:.3e}")
    assert np.isfinite(mse) and mse < mse_tol and rel < rel_tol, f"{name}: mse={mse:.3e} rel_rms={rel:.3e}"


def _assert_fp16_of(got, ref64):
    """got (fp16) is ref64 rounded once to fp16: within one fp16 ulp of the float64 value."""
    g, r = got.double().cpu(), ref64.double().cpu()
    ulp = torch.clamp(r.abs(), min=2.0 ** -14) * 2.0 ** -10
    assert ((g - r).abs() <= ulp).all(), ((g - r).abs() / ulp).max().item()


# ----------------------------------------------------------------------------------------------- update kernel
@pytest.mark.parametrize("kind,eta", [("euler_a", 1.0), ("euler_a", 0.0), ("dpmpp_2m", 0.0)])
@pytest.mark.parametrize("cfg", [True, False])
def test_update_kernel_matches_float64(kind, eta, cfg):
    from oracle import pfd_oracle as PO
    from pfd_b200 import native as nv
    from pfd_b200 import sampler as S
    dev = "cuda"
    n = 6
    sig = S.get_sigmas(PO.schedule_buffers()["alphas_cumprod"].half(), n).double().numpy()
    coef = torch.as_tensor(S.coef_table(kind, sig, eta), dtype=torch.float32)
    g = torch.Generator().manual_seed(5)
    B, shape = 2, (2, 4, 9, 7)
    half_n = int(np.prod(shape))
    guidance = 2.5 if cfg else 1.5
    for k in (0, 2, n - 1):
        for with_noise in (False, True):
            eps = torch.randn(((2 if cfg else 1) * B,) + shape[1:], generator=g).half()
            x = torch.randn(shape, generator=g) * float(sig[k])
            dprev = torch.randn(shape, generator=g)
            noise = torch.randn(shape, generator=g).half() if with_noise else None
            xd, dd = x.to(dev), dprev.to(dev)
            uin = torch.full(eps.shape, 7.0, dtype=torch.float16, device=dev)
            out = torch.full(shape, 7.0, dtype=torch.float16, device=dev)
            log_tab = torch.full((n,), -1, dtype=torch.int32)
            log_tab[k] = 1
            log_xt = torch.zeros((2,) + shape, dtype=torch.float16, device=dev)
            log_x0 = torch.zeros_like(log_xt)
            step = torch.tensor([k], dtype=torch.int32, device=dev)
            nv.ksampler_step(eps.to(dev), cfg, guidance, coef.to(dev), step, n - 1, xd, dd, uin, out,
                             noise=None if noise is None else noise.to(dev), log_tab=log_tab.to(dev),
                             log_xt=log_xt, log_x0=log_x0)
            torch.cuda.synchronize()
            # float64 restatement with the fp32 table values
            s_, a, b, c, u, cn = (float(v) for v in coef[k])
            e64 = eps.double()
            e = (e64[:B] + guidance * (e64[B:] - e64[:B])) if cfg else guidance * e64
            x64 = x.double()
            d = x64 - s_ * e
            xn = a * x64 + b * d + c * dprev.double()
            if noise is not None:
                xn = xn + u * noise.double()
            scale = xn.abs().max().item() + 1.0
            assert (xd.double().cpu() - xn).abs().max().item() < 2e-6 * scale, (k, with_noise)
            assert (dd.double().cpu() - d).abs().max().item() < 2e-6 * (d.abs().max().item() + 1.0)
            _assert_fp16_of(uin[:B], xn * cn)
            if cfg:
                assert torch.equal(uin[:B], uin[B:])
            if k == n - 1:
                _assert_fp16_of(out, xn)
            else:
                assert (out == 7.0).all()
            assert torch.equal(log_xt[1], uin[:B]) and (log_xt[0] == 0).all()
            _assert_fp16_of(log_x0[1], d)


# ----------------------------------------------------------------------------------------------- embedding
def test_float_timestep_embedding():
    from pfd_b200 import native as nv
    dim = 320
    t = torch.tensor([0.0, 0.37, 1.0, 12.5, 501.0, 947.421, 998.99, 999.0], device="cuda")
    emb = nv.timestep_embedding(t, dim)
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64) / half)
    args = t.double().cpu()[:, None] * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    assert (emb.double().cpu() - ref).abs().max().item() < 2e-3
    ti = torch.arange(0, 1000, 7, device="cuda")
    assert torch.equal(nv.timestep_embedding(ti.float(), dim), nv.timestep_embedding(ti, dim))
    assert torch.equal(nv.timestep_embedding(ti.float(), 321), nv.timestep_embedding(ti, 321))
    with pytest.raises(RuntimeError):
        nv.timestep_embedding(ti.int(), dim)


# ----------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def env():
    from oracle.golden_inputs import golden_inputs
    from pfd_b200 import get_model, model_cfg_bank
    from pfd_b200.weights import SCHEDULE_BUFFERS, fill_module_
    net = get_model()(model_cfg_bank()("pfd_seecoder_with_controlnet"))
    fill_module_(net, seed=0, skip=SCHEDULE_BUFFERS)
    net = net.half()
    net.to("cuda")
    net.eval()
    inp = {k: v.cuda() for k, v in golden_inputs().items()}
    return net, inp


def _c_info(inp, control, guidance=2.0):
    cond = inp["cond"].half()
    return {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
            "unconditional_guidance_scale": guidance, "control": inp["hint"].half() if control else None}


def _oracle_denoiser(net, inp, control, guidance=2.0):
    """D(x, sigma) = x - sigma * CFG(eps) with eps from the torch oracle of the UNet (+ ControlNet) in fp16 on the GPU,
    evaluated at the fp16 UNet input x*c_in and the float timestep t(sigma)."""
    from oracle import pfd_oracle as PO
    from pfd_b200 import sampler as S
    sd = {k: v.detach() for k, v in net.state_dict().items()}
    usd = PO.sub(sd, "diffuser.image.")
    csd = PO.sub(sd, "ctl.")
    ls = S.model_log_sigmas(net.alphas_cumprod)
    cond = inp["cond"].half()
    c_in = torch.cat([torch.zeros_like(cond), cond])
    hint = inp["hint"].half()

    def eps_of(xin, t):
        xx = torch.cat([xin, xin])
        tt = torch.full((xx.shape[0],), t, dtype=torch.float32, device=xin.device)
        ctl = PO.controlnet_apply(csd, PO.CONTROLNET_SD15, xx, hint, tt, c_in) if control else None
        e = PO.unet_apply(usd, PO.UNET_SD15, xx, tt, c_in, ctl).double()
        eu, ec = e.chunk(2)
        return eu + guidance * (ec - eu)

    def denoise_input(xin, sigma):
        """teacher forcing: the fp16 UNet input the sampler produced -> D"""
        t = float(S.sigma_to_t([sigma], ls)[0])
        cin = 1.0 / math.sqrt(sigma * sigma + 1.0)
        return xin.double() / cin - sigma * eps_of(xin, t)

    def denoise(x, sigma):
        cin = 1.0 / math.sqrt(sigma * sigma + 1.0)
        return denoise_input((x * cin).half(), sigma)
    return denoise, denoise_input


@pytest.mark.parametrize("kind,control", [("dpmpp_2m", True), ("euler_a", False)])
def test_sampler_matches_oracle_loop(env, kind, control):
    net, inp = env
    from oracle import sampler_oracle as SO
    from pfd_b200 import Sampler
    steps, seed = 8, 31
    xt = inp["x_T"].half()
    torch.manual_seed(seed)
    x, inter = Sampler(net, type=kind).sample(steps=steps, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": xt},
                                              c_info=_c_info(inp, control), log_every_t=1)
    assert x.dtype == torch.float16 and x.shape == (1, 4, 16, 16)
    assert len(inter["pred_xt"]) == len(inter["pred_x0"]) == steps
    assert torch.equal(inter["pred_xt"][-1], x)
    sig = Sampler(net).get_sigmas(steps).double().numpy()
    eta = 1.0 if kind == "euler_a" else 0.0
    denoise, denoise_input = _oracle_denoiser(net, inp, control)
    with torch.no_grad():
        # per evaluation, teacher-forced on the sampler's own fp16 UNet inputs
        cin0 = 1.0 / math.sqrt(sig[0] ** 2 + 1.0)
        xin = (xt.float() * float(sig[0]) * cin0).half()
        for k in range(steps):
            _check(f"{kind} D at step {k} (teacher-forced)", inter["pred_x0"][k], denoise_input(xin, float(sig[k])),
                   rel_tol=5e-3)
            xin = inter["pred_xt"][k]
        # free-running float64 oracle loop on the same x_T and noise stream
        torch.manual_seed(seed)
        noises = [torch.randn((1, 4, 16, 16), device="cuda", dtype=torch.float16) if (eta and sig[k + 1] > 0) else None
                  for k in range(steps)]
        ref = SO.run_table(denoise, xt.double() * float(sig[0]), SO.coef_table(kind, sig, eta), noises)
    _check(f"{kind} final latent ({'control' if control else 'plain'})", x, ref, rel_tol=2e-2)


def test_euler_on_ddim_timesteps_reproduces_ddim(env):
    """Plain Euler in sigma is DDIM (eta 0) in x / sqrt(alpha_bar): same steps, same UNet evaluations."""
    net, inp = env
    from pfd_b200 import DDIMSampler, Sampler
    from pfd_b200 import sampler as S
    from pfd_b200.ddim import make_ddim_timesteps
    steps = 4
    ts = make_ddim_timesteps(steps, 1000)                               # [1, 251, 501, 751]
    ls = S.model_log_sigmas(net.alphas_cumprod).double()
    sig = [math.exp(float(ls[int(t)])) for t in ts[::-1]] + [math.exp(float(ls[0]))]
    x_T = inp["x_T"].half()
    xd, _ = DDIMSampler(net).sample(steps=steps, x_info={"type": "image", "xt": x_T}, c_info=_c_info(inp, False),
                                    shape=[1, 4, 16, 16], verbose=False, eta=0.0)
    cin = lambda s: 1.0 / math.sqrt(s * s + 1.0)
    xt = x_T.float() / (sig[0] * cin(sig[0]))                           # sigma_0 * xt * c_in(sigma_0) == x_T
    xs, _ = Sampler(net, type="euler_a").sample(steps=None, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": xt},
                                                c_info=_c_info(inp, False), eta=0.0, sigmas=sig)
    _check("euler (eta 0) on DDIM timesteps vs DDIM", xs.float() * cin(sig[-1]), xd, rel_tol=2e-2)


# ----------------------------------------------------------------------------------------------- graphs
def _run(sampler, inp, seed, control=False, **kw):
    torch.manual_seed(seed)
    x, _ = sampler.sample(steps=kw.pop("steps", 6), shape=[1, 4, 16, 16], x_info={"type": "image"},
                          c_info=_c_info(inp, control), **kw)
    return x


def test_graphs_match_eager_and_follow_weight_swaps(env):
    net, inp = env
    from pfd_b200 import Sampler
    # GroupNorm statistics are combined with fp64 atomics, so replays agree to rounding, not bit for bit
    tol = 5e-3
    for kind, eta, control in (("dpmpp_2m", 0.0, True), ("euler_a", 1.0, False)):
        g = Sampler(net, type=kind)
        e = Sampler(net, type=kind, use_cuda_graph=False)
        a1, a2 = _run(g, inp, 5, control, eta=eta), _run(g, inp, 5, control, eta=eta)
        b = _run(e, inp, 5, control, eta=eta)
        _check(f"{kind} graph replay vs first call", a2, a1, rel_tol=tol)
        _check(f"{kind} graph vs eager", a1, b, rel_tol=tol)
        other = _run(g, inp, 6, control, eta=eta)
        assert (other.float() - a1.float()).abs().max().item() > 0.1   # seed-dependent
    # hot swap of the diffuser weights: the cached graph must not replay stale weights
    s = Sampler(net, type="dpmpp_2m")
    base = _run(s, inp, 9)
    orig = {k: v.detach().clone() for k, v in net.diffuser.state_dict().items()}
    mod = dict(orig)
    mod["image.data_blocks.0.0.weight"] = orig["image.data_blocks.0.0.weight"] * 1.5    # the UNet's conv_in
    net.diffuser.load_state_dict(mod)
    try:
        swapped = _run(s, inp, 9)
    finally:
        net.diffuser.load_state_dict(orig)
    restored = _run(s, inp, 9)
    assert (swapped.float() - base.float()).pow(2).mean().sqrt().item() > 0.05 * base.float().pow(2).mean().sqrt().item()
    _check("dpmpp_2m after restoring the weights", restored, base, rel_tol=tol)
