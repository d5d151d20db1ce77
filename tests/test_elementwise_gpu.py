"""Exact checks of the elementwise kernels (pfd_b200/csrc/elementwise.cu) and of the activations of the GEMM epilogue.

Where the contract is a single fp16 rounding the comparison is on bits: the DDIM update against the reference step
evaluated in eager torch fp16 (elementwise_ref.ddim_eager), the VAE posterior's mean / logvar, the Swin and layout
kernels, add_rowvec, axpby with unit scales, ReLU.  Where an fp32 approximation is involved (the timestep embedding's
libm chain, __expf in the posterior and SiLU, fast_erf, gelu_sig, axpby's fused multiply-add) the bound is derived
beside the check.  The activations run over all 63 488 finite fp16 pre-activations, on the staged, the split-K and
the element-strided epilogue routes.
"""
import numpy as np
import pytest
import torch

from attention_ref import ulp16
from elementwise_ref import (DDIM_GUIDANCE_CFG, DDIM_GUIDANCE_NOCFG, DDIM_STEPS, DDIM_TEMPERATURES,
                             WINDOW_GEOMETRIES, WINDOW_SIZES, all_finite_f16, bit_mismatch, bits, ddim_coefs,
                             ddim_eager, ddim_inputs, ddim_schedule_sampler, geglu_gate_errors, gelu64,
                             gelu_sig_bound, half_rn, padded, temb_ref, window_gather_ref, window_scatter_ref)
from test_gemm_paths_gpu import layout

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


def grid_cap():
    """Elements one grid_for() launch covers in one grid-stride pass (16 CTAs of 256 threads per SM)."""
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * 256


def rnd(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to("cuda", dtype)


def assert_bits(out, ref, what):
    bad = bits(out) != bits(ref)
    assert not bad.any(), (f"{what}: {bad.sum().item()}/{bad.numel()} elements differ, e.g. "
                           f"{out.reshape(-1)[bad.reshape(-1)][:4].tolist()} vs {ref.reshape(-1)[bad.reshape(-1)][:4].tolist()}")


def assert_within(out, ref, tol, what):
    err = (out.double() - ref.double()).abs()
    bad = err > tol
    assert not bad.any(), (f"{what}: {bad.sum().item()}/{bad.numel()} outside the bound, max err/bound "
                           f"{(err / tol).max().item():.3g}")


# ================================================================================================ 1. DDIM update
@pytest.fixture(scope="module")
def samplers():
    return {eta: ddim_schedule_sampler(eta) for eta in (0.0, 1.0)}


DDIM_SIZES = {"latent512_b2": (2, 4, 64, 64), "ragged": (2, 4, 13, 7), "above_grid_cap": (8, 4, 192, 192)}


def ddim_run(nv, eps, x, guidance, coef, step, noise, temperature, inplace, log=None):
    if inplace:                                     # x_prev is x, as _DDIMState calls it
        xp = x.clone()
        src = xp
    else:
        xp, src = torch.empty_like(x), x
    p0 = torch.empty_like(x)
    kw = {} if log is None else dict(log_tab=log[0], log_xt=log[1], log_x0=log[2])
    nv.ddim_step(eps, src, guidance, coef, step, xp, p0, noise=noise, temperature=temperature, **kw)
    return xp, p0


@pytest.mark.parametrize("size", list(DDIM_SIZES))
@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_ddim_step_bitwise(nv, samplers, eta, size):
    """Every schedule index (through the device step pointer) x guidance (CFG and not) x temperature x noise x input
    scale; x_prev and pred_x0 bit for bit against the eager fp16 reference step."""
    smp = samplers[eta]
    assert np.prod(DDIM_SIZES["above_grid_cap"]) > grid_cap()
    shape = DDIM_SIZES[size]
    coef = smp._coef_table("cuda")
    steps = torch.arange(DDIM_STEPS, dtype=torch.int32, device="cuda")
    # log slots: every 7th index logged, the others -1
    log_tab = torch.tensor([i // 7 if i % 7 == 0 else -1 for i in range(DDIM_STEPS)], dtype=torch.int32,
                           device="cuda")
    nslots = (DDIM_STEPS + 6) // 7
    failures = []
    for scale in (1.0, 30.0):
        for guidance in DDIM_GUIDANCE_CFG + DDIM_GUIDANCE_NOCFG:
            cfg = guidance not in DDIM_GUIDANCE_NOCFG
            eps, x, noise = (t.cuda() for t in ddim_inputs(shape, scale, seed=int(guidance * 10) + int(scale),
                                                             cfg=cfg))
            for index in range(DDIM_STEPS):
                c = ddim_coefs(smp, index, False, "cuda", x.dim())
                step = steps[index:index + 1]
                for k, (temperature, nz) in enumerate((t, n) for t in DDIM_TEMPERATURES for n in (noise, None)):
                    xp_r, p0_r = ddim_eager(eps, x, guidance, c, nz, temperature, cfg)
                    log = None
                    if k == 0:
                        log = (log_tab, torch.full((nslots,) + shape, float("nan"), device="cuda",
                                                   dtype=torch.float16),
                               torch.full((nslots,) + shape, float("nan"), device="cuda", dtype=torch.float16))
                    xp, p0 = ddim_run(nv, eps, x, guidance, coef, step, nz, temperature, inplace=k % 2 == 0, log=log)
                    n_xp, n_p0 = int(bit_mismatch(xp, xp_r).sum()), int(bit_mismatch(p0, p0_r).sum())
                    if n_xp or n_p0:
                        failures.append(f"scale {scale} g {guidance} index {index} T {temperature} noise "
                                        f"{nz is not None}: {n_xp} x_prev / {n_p0} pred_x0")
                    if log is not None:
                        slot = int(log_tab[index])
                        for buf, want in ((log[1], xp), (log[2], p0)):
                            for s in range(nslots):
                                if s == slot:
                                    assert not bit_mismatch(buf[s], want).any(), f"index {index}: log slot {s}"
                                else:
                                    assert torch.isnan(buf[s]).all(), f"index {index}: slot {s} written"
    assert not failures, f"{len(failures)} cases differ, e.g. " + "; ".join(failures[:6])


@pytest.mark.parametrize("eta", [0.0, 1.0])
def test_ddim_step_original_steps(nv, samplers, eta):
    """step = None with the one-row table of _coef_original (use_original_steps, ddim.py:150-153)."""
    smp = samplers[eta]
    shape = (2, 4, 13, 7)
    for guidance in (7.5, 1.0):
        cfg = guidance != 1.0
        eps, x, noise = (t.cuda() for t in ddim_inputs(shape, 1.0, seed=11, cfg=cfg))
        for index in (1, 2, 10, 100, 333, 500, 750, 999):
            coef = smp._coef_original(index).cuda()
            c = ddim_coefs(smp, index, True, "cuda", x.dim())
            for temperature, nz in ((1.0, None), (0.7, noise), (0.9, noise)):
                xp_r, p0_r = ddim_eager(eps, x, guidance, c, nz, temperature, cfg)
                xp, p0 = ddim_run(nv, eps, x, guidance, coef, None, nz, temperature, inplace=True)
                assert not bit_mismatch(xp, xp_r).any(), f"index {index} T {temperature}: x_prev"
                assert not bit_mismatch(p0, p0_r).any(), f"index {index} T {temperature}: pred_x0"


def test_ddim_begin_step_walks_and_stops_at_zero(nv):
    total, nb = DDIM_STEPS, 130                     # nb > the header's 64 threads
    ttab = torch.tensor(np.arange(total) * 20 + 1, dtype=torch.int64, device="cuda")
    step = torch.full((1,), total, dtype=torch.int32, device="cuda")
    t_out = torch.full((nb,), -5, dtype=torch.int64, device="cuda")
    for i in range(total):
        nv.ddim_begin_step(step, ttab, t_out)
        s = int(step)
        assert s == total - 1 - i
        assert (t_out == ttab[s]).all(), f"call {i}: t_out {t_out.unique().tolist()} vs {int(ttab[s])}"
    nv.ddim_begin_step(step, ttab, t_out)           # one call too many: the counter stays at 0
    assert int(step) == 0 and (t_out == ttab[0]).all()


# ================================================================================================ 2. timestep embedding
@pytest.mark.parametrize("dim", [320, 321])
@pytest.mark.parametrize("max_period", [10000.0, 1000.0])
def test_timestep_embedding(nv, dim, max_period):
    # every integer timestep, 16 per call (the largest batch of timesteps the pipelines embed at once)
    t_int = torch.arange(1000, dtype=torch.int64)
    g = torch.Generator().manual_seed(dim)
    t_frac = (torch.rand(1000, generator=g, dtype=torch.float64) * 999).float()
    for name, t in (("int64", t_int), ("float32", t_frac)):
        outs = [nv.timestep_embedding(t[i:i + 16].cuda(), dim, max_period) for i in range(0, 1000, 16)]
        out = torch.cat(outs).double().cpu()
        ref, bound = temb_ref(t.double(), dim, max_period)
        err = (out - ref).abs()
        assert (err <= bound).all(), f"{name}: max err/bound {(err / bound.clamp_min(1e-30)).max().item():.3g}"
        if dim % 2:
            assert (bits(torch.cat(outs)[:, -1]) == 0).all(), f"{name}: last column not +0"
    # the float32 entry point at integer t: the same bits as the int64 one
    for n in (1, 7, 16):
        ti = torch.tensor([0, 1, 999, 981, 500, 21, 2, 998, 3, 4, 5, 6, 7, 8, 9, 10][:n], dtype=torch.int64)
        assert_bits(nv.timestep_embedding(ti.float().cuda(), dim, max_period),
                    nv.timestep_embedding(ti.cuda(), dim, max_period), f"float32 vs int64 entry, n={n}")


# ================================================================================================ 3. VAE posterior
LOGVAR_EDGES = (-65504.0, -31.0, -30.0, -29.98, 19.98, 20.0, 21.0, 65504.0)
OUTPUT_SETS = [tuple(k for j, k in enumerate(("mean", "logvar", "std", "sample")) if m >> j & 1) for m in range(1, 16)]


@pytest.mark.parametrize("B,H,W", [(1, 64, 64), (2, 96, 96), (1, 192, 192), (2, 13, 7)])
def test_vae_posterior(nv, B, H, W):
    zc, cpad = 4, 8                                   # autokl.py: quant_conv gives 2 * zc = 8 channel-last moments
    g = torch.Generator().manual_seed(H * W + B)
    mom = torch.randn((B, H, W, cpad), generator=g) * 3
    lv = (torch.randn((B, H, W, zc), generator=g) * 8 - 4).reshape(-1)
    lv[0::2] = torch.tensor(LOGVAR_EDGES).repeat(lv.numel() // 2 // len(LOGVAR_EDGES) + 1)[:lv[0::2].numel()]
    mom[..., zc:2 * zc] = lv.reshape(B, H, W, zc)
    mom = mom.half().cuda()
    assert all((mom[..., zc:2 * zc] == e).any() for e in LOGVAR_EDGES)
    noise = torch.randn((B, zc, H, W), generator=g).cuda()
    mu_ref = mom[..., :zc].permute(0, 3, 1, 2)
    lv_ref = mom[..., zc:2 * zc].permute(0, 3, 1, 2).clamp(-30.0, 20.0)
    for scale in (1.0, 0.18215):
        for nz in (noise, None):
            o = nv.vae_posterior(mom, zc, noise=nz, scale=scale)
            assert_bits(o["mean"], mu_ref.contiguous(), "mean")
            assert_bits(o["logvar"], lv_ref.contiguous(), "logvar")
            # __expf: a few fp32 ulps, then one fp16 rounding -> within one ulp of the correctly rounded value
            std64 = torch.exp(0.5 * lv_ref.double())
            assert_within(o["std"], half_rn(std64), ulp16(std64), "std")
            # sample = fp16(scale * fmaf(std, noise, mu)) with the kernel's fp16 std: two fp32 roundings and one fp16
            ref = float(np.float32(scale)) * (mu_ref.double() + o["std"].double() * (0 if nz is None else nz.double()))
            out = o["sample"].double()
            ovf = ref.abs() >= 65520                          # beyond the fp16 range: inf of the same sign
            assert (out[ovf] == torch.sign(ref[ovf]) * float("inf")).all()
            assert_within(out[~ovf], ref[~ovf], ulp16(ref[~ovf]), f"sample scale {scale} noise {nz is not None}")
    full = nv.vae_posterior(mom, zc, noise=noise, scale=0.18215)
    for want in OUTPUT_SETS:
        o = nv.vae_posterior(mom, zc, noise=noise, scale=0.18215, want=want)
        assert set(o) == set(want)
        for k in want:
            assert_bits(o[k], full[k], f"{k} of {want}")


# ================================================================================================ 4. Swin / SeeCoder
@pytest.mark.parametrize("H,W,C", WINDOW_GEOMETRIES)
def test_window_gather_scatter(nv, H, W, C):
    B = 2 if H * W * C <= 64 * 64 * 384 else 1
    x = rnd((B, H, W, C), H * W + C)
    res = rnd((B, H, W, C), H * W + C + 1, 4.0)
    for ws in WINDOW_SIZES:
        for shift in (0, ws // 2):
            tag = f"ws {ws} shift {shift}"
            win = nv.window_gather(x, ws, shift)
            assert_bits(win, window_gather_ref(x, ws, shift), f"gather {tag}")
            Hp, Wp = padded(H, W, ws)
            ids = torch.arange(1, B * H * W + 1, dtype=torch.float64).reshape(B, H, W, 1)
            pad = window_gather_ref(ids, ws, shift)[..., 0] == 0
            if Hp > H or Wp > W:
                assert pad.any()
            assert (bits(win)[pad.cuda()] == 0).all(), f"pad tokens of {tag} not +0"
            w2 = rnd(win.shape, H + W + ws + shift)
            assert_bits(nv.window_scatter(w2, B, H, W, ws, shift, None), window_scatter_ref(w2, B, H, W, ws, shift),
                        f"scatter {tag}")
            ref = half_rn(window_scatter_ref(w2, B, H, W, ws, shift).double() + res.double())
            assert_bits(nv.window_scatter(w2, B, H, W, ws, shift, res), ref, f"scatter + residual {tag}")
            assert_bits(nv.window_scatter(win, B, H, W, ws, shift, None), x, f"scatter(gather) {tag}")


@pytest.mark.parametrize("H,W,C", [(128, 128, 192), (13, 29, 384), (7, 7, 768), (1, 3, 1536), (64, 64, 384)])
def test_patch_merge_gather(nv, H, W, C):
    x = rnd((2, H, W, C), H * W)
    xp = torch.nn.functional.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    ref = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1)
    assert_bits(nv.patch_merge_gather(x), ref, "patch merge")


@pytest.mark.parametrize("C,P,H,W,kpad", [(3, 4, 64, 64, 48), (3, 4, 66, 70, 48), (3, 3, 31, 29, 32),
                                          (1, 4, 17, 9, 24)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_patchify(nv, C, P, H, W, kpad, dtype):
    img = rnd((2, C, H, W), H * W + P, 2.0, torch.float32).to(dtype)
    Hq, Wq = -(-H // P), -(-W // P)
    xp = torch.nn.functional.pad(img.double(), (0, Wq * P - W, 0, Hq * P - H))
    cols = xp.reshape(2, C, Hq, P, Wq, P).permute(0, 2, 4, 1, 3, 5).reshape(2, Hq, Wq, C * P * P)
    ref = torch.nn.functional.pad(cols, (0, kpad - C * P * P)).float().half()  # the fp32 value rounded once
    assert_bits(nv.patchify(img, P, kpad), ref, f"patchify {dtype}")


# ================================================================================================ 5. small kernels
@pytest.mark.parametrize("C", [768, 256])
def test_add_rowvec(nv, C):
    a, row = rnd((1000, C), C, 8.0), rnd((C,), C + 1, 8.0)
    ref = half_rn(a.double() + row.double())
    assert_bits(nv.add_rowvec(a, row), ref, "add_rowvec")
    nv.add_rowvec(a, row, out=a)                         # in place, as seecoder.py:98 calls it
    assert_bits(a, ref, "add_rowvec in place")


@pytest.mark.parametrize("n", [1000, 2 * 540672 + 37])
def test_axpby(nv, n):
    a, b = rnd((n,), n, 4.0), rnd((n,), n + 1, 4.0)
    # unit scales (the ControlNet residual add): one rounding of the exact sum
    assert_bits(nv.axpby(a, 1.0, b, 1.0), half_rn(a.double() + b.double()), "axpby(1, 1)")
    # fp32 scales (q_sample, axpby(x0, sqrt(a_t), noise, sqrt(1 - a_t))): fma(b, sb, fp32(a * sa)) rounds to fp32
    # twice (2^-24 of |a * sa| and of the result) and once to fp16, where the reference rounds a * sa and b * sb to
    # fp16 first (unet.py:401).  Bound: one fp16 ulp plus the two fp32 roundings, which matter only where the two
    # products cancel
    u = 2.0 ** -24
    for sa, sb in ((0.9183, 0.3959), (0.0683, 0.9977), (-1.7, 2.3)):
        sa32, sb32 = float(np.float32(sa)), float(np.float32(sb))
        ref = a.double() * sa32 + b.double() * sb32
        tol = ulp16(ref) + u * ((a.double() * sa32).abs() + ref.abs())
        assert_within(nv.axpby(a, sa, b, sb), ref, tol, f"axpby({sa}, {sb})")
        ref = a.double() * sa32
        assert_within(nv.axpby(a, sa), ref, ulp16(ref) + u * ref.abs(), f"axpby({sa}, b=None)")
    if n > grid_cap():
        assert_bits(nv.axpby(a, 1.0, b, 1.0)[-37:], half_rn(a[-37:].double() + b[-37:].double()), "tail")


@pytest.mark.parametrize("C", [320, 640, 1280])
def test_upsample2x(nv, C):
    x = rnd((2, 9, 13, C), C)
    assert_bits(nv.upsample2x(x), x.repeat_interleave(2, 1).repeat_interleave(2, 2), "upsample2x")


def test_nchw_to_nhwc(nv):
    g = torch.Generator().manual_seed(0)
    x = torch.rand((2, 3, 37, 41), generator=g).cuda()   # multiples of 2^-24 in [0, 1): 2x - 1 is exact in float64
    # the VAE input 2x - 1 (fp32 source): fp16(fmaf(x, 2, -1)), padded 3 -> 8 channels with zeros
    ref = torch.nn.functional.pad((x.double() * 2 - 1).float().permute(0, 2, 3, 1), (0, 5)).half()
    out = nv.nchw_to_nhwc(x, cpad=8, mul=2.0, add=-1.0)
    assert_bits(out, ref, "nchw_to_nhwc fp32 2x-1")
    xh = rnd((2, 5, 7, 9), 3)
    assert_bits(nv.nchw_to_nhwc(xh, cpad=8), torch.nn.functional.pad(xh.permute(0, 2, 3, 1), (0, 3)), "fp16 copy")


def test_nhwc_to_nchw(nv):
    x = rnd((2, 21, 19, 8), 4, 1.5)
    # the VAE output (x + 1) / 2 clamped to [0, 1] from 4 of 8 channels: x * 0.5 + 0.5 is exact, rounded once
    out = nv.nhwc_to_nchw(x, 4, mul=0.5, add=0.5, lo=0.0, hi=1.0)
    ref = half_rn(x[..., :4].double() * 0.5 + 0.5).double().clamp(0.0, 1.0).half().permute(0, 3, 1, 2)
    assert ((ref == 0) | (ref == 1)).any()
    assert_bits(out, ref.contiguous(), "nhwc_to_nchw")


@pytest.mark.parametrize("H,W,C,stride,kpad", [(33, 17, 3, 2, 32), (9, 7, 4, 2, 40), (16, 12, 8, 1, 72),
                                               (5, 5, 3, 1, 32)])
def test_im2col3x3(nv, H, W, C, stride, kpad):
    x = rnd((2, H, W, C), H * W + C)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    taps = [xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
            for ky in range(3) for kx in range(3)]
    ref = torch.nn.functional.pad(torch.cat(taps, -1), (0, kpad - 9 * C))
    assert_bits(nv.im2col3x3(x, kpad, stride), ref, "im2col3x3")


# ================================================================================================ 6. epilogue activations
def act_values():
    g = all_finite_f16()
    assert g.numel() == 63488
    return g


def act_operands(g, K):
    """A [M, K] with g in column 0 (the rest 0) and B = e_0: the accumulator is g exactly."""
    a = torch.zeros((g.numel(), K), dtype=torch.float16)
    a[:, 0] = g
    return a.cuda()


ROUTES = {
    # route: (K, rows per call, N, output layout, kernel launches per call)
    "staged": (64, 63488, 64, "nhwc", 1),
    "element_strided": (64, 63488, 64, "nchw", 1),
    "splitk_finish": (5120, 256, 328, "nhwc", 2),
}


def run_act(nv, a, N, K, kind, act):
    M = a.shape[0]
    w = torch.zeros((N, K), dtype=torch.float16, device="cuda")
    w[:, 0] = 1
    shape, so, ndiv, cdiv, canon = layout(kind, 1, 1, M, N)
    out = torch.empty(shape, device="cuda", dtype=torch.float16)
    n0 = nv.launch_count()
    nv.gemm_raw([(a, 1, K, (K, K * M, K * M))], in_w=M, in_h=1, stride=1, W=M, H=1, NB=1, w=w, N=N, K=K,
                act=act, out=out, so=so, ndiv=ndiv, cdiv=cdiv)
    return canon(out).reshape(M, N), nv.launch_count() - n0


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("act", ["silu", "gelu", "relu"])
def test_epilogue_activation_every_fp16(nv, act, route):
    import pfd_b200
    K, rows, N, kind, launches = ROUTES[route]
    code = {"silu": nv.ACT_SILU, "gelu": nv.ACT_GELU, "relu": nv.ACT_RELU}[act]
    g = act_values()
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(False)
    try:
        outs = []
        a = act_operands(g[:rows], K)
        for i in range(0, g.numel(), rows):
            gi = g[i:i + rows]
            if i:
                a[:gi.numel(), 0] = gi.cuda()
            o, n = run_act(nv, a[:gi.numel()] if gi.numel() < rows else a, N, K, kind, code)
            assert n == launches, f"{route}: {n} kernel launches, expected {launches}"
            outs.append(o[:, :8].clone())
        out = torch.cat(outs)
    finally:
        pfd_b200.set_deterministic(was)
    assert (bits(out) == bits(out[:, :1])).all(), "columns of one row differ"
    out = out[:, 0].double().cpu()
    v = g.double()
    if act == "relu":
        # exact; compared as values because the accumulator of g = -0 is +0 (-0 + 0 products), so its sign is not g's
        bad = out != v.clamp(min=0)
        assert not bad.any(), f"relu: {int(bad.sum())} outputs differ, e.g. at g = {v[bad][:4].tolist()}"
        return
    ref = v * torch.sigmoid(v) if act == "silu" else gelu64(v)
    # one fp16 ulp (fp32 approximations near a rounding boundary); GELU adds fast_erf's 1.5e-7 absolute error times
    # |v| / 2 (1 + erf cancels for v << 0), the contract of test_gemm_paths_gpu.py
    tol = ulp16(torch.maximum(out.abs(), ref.abs()))
    if act == "gelu":
        tol = tol + 2e-7 * v.abs()
    assert_within(out, ref, tol, f"{act} on {route}")


GEGLU_VALUES = (1.0, 0.75, -3.0, 2.0 ** -10)


def test_geglu_every_fp16_gate(nv):
    """GEGLU through pack_geglu: A rows [g, 1, 0, ...]; value rows of the weight pick column 1 times a value operand,
    gate rows pick column 0, so value = v and gate = g exactly and out = fp16(v * fp16(gelu_sig(g))) (__hmul2)."""
    g = act_values()
    K, inner = 64, 64
    a = act_operands(g, K)
    a[:, 1] = 1
    w = torch.zeros((2 * inner, K), dtype=torch.float16)
    w[:inner, 1] = torch.tensor(GEGLU_VALUES, dtype=torch.float16).repeat(inner // len(GEGLU_VALUES))
    w[inner:, 0] = 1
    wp, bp, _ = nv.pack_geglu(w.cuda(), None)
    n0 = nv.launch_count()
    out = nv.linear(a, wp, bp, act=nv.ACT_GEGLU)
    assert nv.launch_count() - n0 == 1
    out = out.cpu()
    gate = out[:, 0]                                    # v = 1: fp16(gelu_sig(g)) itself
    err = geglu_gate_errors(gate, g)
    off = int((bits(gate) != bits(half_rn(gelu64(g)))).sum())
    print(f"[geglu] gate max err/bound {err.max().item():.3f}; {off} of {g.numel()} gates differ from "
          f"correctly rounded GELU")
    assert (err <= 1).all(), f"{int((err > 1).sum())} gates outside the bound"
    for j, v in enumerate(GEGLU_VALUES):
        col = out[:, j]
        assert_bits(col, half_rn(v * gate.double()), f"value {v}: fp16(v * gate)")
        # against float64 v * gelu(g): the two roundings plus |v| times the gelu_sig bound; products beyond the fp16
        # range (v = -3, g > 21840) must be inf of the right sign
        ref = v * gelu64(g)
        ovf = ref.abs() >= 65520
        assert (col[ovf].double() == torch.sign(ref[ovf]) * float("inf")).all(), f"value {v}: overflow"
        col, ref, gv, gg = col[~ovf], ref[~ovf], gate[~ovf].double(), g[~ovf]
        tol = 0.5 * ulp16(torch.maximum(col.double().abs(), ref.abs())) + abs(v) * (
            0.5 * ulp16(gv) + gelu_sig_bound(gg))
        assert_within(col, ref, tol, f"value {v} vs float64")
    assert all(torch.equal(bits(out[:, j]), bits(out[:, j % len(GEGLU_VALUES)])) for j in range(inner))
