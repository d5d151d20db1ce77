"""Deterministic mode (pfd_b200.set_deterministic): every output is a bitwise function of the sample's own inputs.
GroupNorm against float64 and bit for bit across calls, batch positions and planning SM counts; the GEMM across forced N
tile widths and across M; the pipeline (SeeCoder context, UNet + ControlNet, DDIM / dpmpp_2m / euler_a, VAE decode, HED) across
batch compositions, calls, graph replay and processes; the mode switch; the multi-GPU split."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


@pytest.fixture
def det(nv):
    import pfd_b200
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(True)
    yield
    nv.set_env_option("plan_sms", 0)
    pfd_b200.set_deterministic(was)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to("cuda", torch.float16)


def close(out, ref, rtol, atol):
    err = (out.float() - ref.float()).abs()
    bad = (err > atol + rtol * ref.float().abs()).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


def rel_rms(a, b):
    a, b = a.double(), b.double()
    return ((a - b).pow(2).mean() / b.pow(2).mean()).sqrt().item()


def assert_same(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), \
        f"{what}: not bit-identical (max abs diff {(a.float() - b.float()).abs().max().item():.3g})"


# ----------------------------------------------------------------------------------------------- GroupNorm
GN_SHAPES = [  # (H, W, C1, C2, silu)
    (64, 64, 320, 0, True),          # UNet level 1
    (8, 8, 2560, 0, True),           # UNet level 4
    (64, 64, 640, 320, True),        # the 960-channel skip concat
    (256, 256, 128, 0, False),       # VAE decoder, 128 chunks per image
    (37, 37, 320, 0, True),          # HW = 1369 is not a multiple of the chunk
    (20, 20, 96, 0, True),           # 3 channels per group: groups straddle the 8-channel vectors
    (8, 8, 2560, 2560, True),        # rows wider than the CTA: a thread owns several vectors
]


@pytest.mark.parametrize("H,W,C1,C2,silu", GN_SHAPES)
def test_groupnorm_deterministic(nv, det, H, W, C1, C2, silu):
    NB, pos = 5, 3
    x1 = rnd(NB, H, W, C1, scale=2.0) + 0.5
    x2 = rnd(NB, H, W, C2, seed=3) if C2 else None
    C = C1 + C2
    gamma, beta = rnd(C, seed=4) + 1.0, rnd(C, seed=5)

    def gn(a, b):
        nv.gn_reset()
        return nv.groupnorm(a, gamma, beta, 1e-5, silu=silu, x2=b)

    out5 = gn(x1, x2)
    xc = x1 if x2 is None else torch.cat([x1, x2], 3)
    ref = F.group_norm(xc.double().permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5)
    if silu:
        ref = F.silu(ref)
    close(out5, ref.permute(0, 2, 3, 1), rtol=6e-3, atol=6e-3)
    assert_same(gn(x1, x2), out5, "repeated call")
    one = gn(x1[pos:pos + 1].contiguous(), None if x2 is None else x2[pos:pos + 1].contiguous())
    assert_same(one[0], out5[pos], "NB = 1 vs position 3 of NB = 5")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for plan in (114, 66):
        nv.set_env_option("plan_sms", plan)
        assert_same(gn(x1, x2), out5, f"plan_sms {plan} vs {sms}")
    nv.set_env_option("plan_sms", 0)


# ----------------------------------------------------------------------------------------------- GEMM
BNS = (64, 128, 160, 192, 256)


def conv3x3(nv, x, wp, b, bn=0):
    NB, H, W, C = x.shape
    N = wp.shape[0]
    out = torch.empty((NB, H, W, N), device="cuda", dtype=torch.float16)
    nv.gemm_raw([(x, 9, C, (x.stride(2), x.stride(1), x.stride(0)))], in_w=W, in_h=H, stride=1, W=W, H=H, NB=NB,
                w=wp, N=N, K=wp.stride(0), bias=b, out=out, so=(out.stride(0), 0, out.stride(1), out.stride(2), 0, 1),
                bn_force=bn)
    return out


def head_split(nv, x, w, b, B, T, heads, d, bn=0):
    out = torch.empty((B, heads, T, d), device="cuda", dtype=torch.float16)
    K = x.shape[1]
    nv.gemm_raw([(x, 1, K, (K, K * T, K * T))], in_w=T, in_h=1, stride=1, W=T, H=1, NB=B, w=w, N=heads * d, K=K,
                bias=b, out=out, so=(heads * T * d, 0, 0, d, T * d, 1), ndiv=1, cdiv=d, bn_force=bn)
    return out


def gemm_case(nv, case):
    """(run(n, bn) -> output of the first n samples, number of samples, samples of the output)"""
    if case == "conv8x8_k23040":                      # output-block conv 2560 -> 1280 at 8x8: split-K by default
        NB, C, N = 5, 2560, 1280
        x, wp, b = rnd(NB, 8, 8, C), rnd(N, 9 * C, scale=(9 * C) ** -0.5, seed=1), rnd(N, seed=2)
        return (lambda n, bn: conv3x3(nv, x[:n], wp, b, bn)), NB, lambda o, i: o[i]
    if case == "linear_residual":                     # proj_out / attention out: K = N = 320, bias + residual
        T, NB = 4096, 5
        x, w, b, r = rnd(NB * T, 320), rnd(320, 320, scale=320 ** -0.5, seed=1), rnd(320, seed=2), rnd(NB * T, 320, seed=3)
        return (lambda n, bn: nv.linear(x[:n * T], w, b, residual=r[:n * T], bn_force=bn)), NB, \
            lambda o, i: o[i * T:(i + 1) * T]
    if case == "geglu":                               # feed-forward GEGLU at the 32x32 level: 640 -> 2 x 2560
        T, NB, C, inner = 1024, 5, 640, 2560
        x, w, b = rnd(NB * T, C), rnd(2 * inner, C, scale=C ** -0.5, seed=1), rnd(2 * inner, seed=2)
        packed = {}

        def run(n, bn):
            bn = bn or nv.geglu_tile(2 * inner)
            if bn not in packed:
                h = bn // 2
                tile = torch.arange(2 * inner // bn, device="cuda").reshape(-1, 1)
                j = torch.arange(h, device="cuda").reshape(1, -1)
                src = torch.stack([tile * h + j, inner + tile * h + j], dim=1).reshape(-1)
                packed[bn] = (w.index_select(0, src).contiguous(), b.index_select(0, src).contiguous())
            wp, bp = packed[bn]
            return nv.linear(x[:n * T], wp, bp, act=nv.ACT_GEGLU, bn_force=bn)
        return run, NB, lambda o, i: o[i * T:(i + 1) * T]
    B, T, heads, d = 5, 1024, 10, 64                  # to_q with a [B, heads, tokens, d] head-split output
    x, w, b = rnd(B * T, 640), rnd(heads * d, 640, scale=640 ** -0.5, seed=1), rnd(heads * d, seed=2)
    return (lambda n, bn: head_split(nv, x[:n * T], w, b, n, T, heads, d, bn)), B, lambda o, i: o[i]


@pytest.mark.parametrize("case", ["conv8x8_k23040", "linear_residual", "geglu", "head_split"])
def test_gemm_tile_width_and_m_invariance(nv, det, case):
    run, NB, sample = gemm_case(nv, case)
    full = run(NB, 0).clone()
    # every N tile width gives the same bits: each output element is accumulated over the same K blocks in order
    for bn in BNS:
        if case == "geglu" and (2 * 2560) % bn:
            continue
        assert_same(run(NB, bn), full, f"{case}: bn_force={bn} vs the library's choice")
    # rows of a small-M product equal the same rows inside the larger product (the planner sees another M)
    for n in (1, 2):
        small = run(n, 0)
        for i in range(n):
            assert_same(sample(small, i), sample(full, i), f"{case}: sample {i} at {n} vs {NB} samples")
    assert_same(sample(run(4, 0), 3), sample(full, 3), f"{case}: sample 3 at 4 vs {NB} samples")


def test_gemm_deterministic_close_to_split_k(nv, det):
    """Deterministic mode turns split-K off; the result stays within rounding of the split-K default."""
    import pfd_b200
    run, NB, _ = gemm_case(nv, "conv8x8_k23040")
    d = run(1, 0).clone()
    pfd_b200.set_deterministic(False)
    s = run(1, 0).clone()
    pfd_b200.set_deterministic(True)
    assert rel_rms(d, s) < 2e-3


# ----------------------------------------------------------------------------------------------- pipeline
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
    inp["xt3"] = torch.cat([seeded((1, 4, 16, 16), 70 + i) for i in range(3)]).cuda().half()
    inp["cond3"] = torch.cat([seeded((1, 148, 768), 80 + i, 0.5) for i in range(3)]).cuda().half()
    return net, inp


def _sample(net, inp, kind, idx, control, graph=True, steps=4):
    from pfd_b200 import DDIMSampler, Sampler
    xt, cond = inp["xt3"][idx], inp["cond3"][idx]
    n = xt.shape[0]
    c_info = {"type": "image", "conditioning": cond, "unconditional_conditioning": torch.zeros_like(cond),
              "unconditional_guidance_scale": 2.0, "control": inp["hint"].half() if control else None}
    shape = [n, 4, 16, 16]
    if kind == "ddim":
        s = DDIMSampler(net, use_cuda_graph=graph)
        x, inter = s.sample(steps=steps, shape=shape, x_info={"type": "image", "xt": xt}, c_info=c_info,
                            verbose=False, eta=0.0, log_every_t=1)
    else:
        s = Sampler(net, type=kind, use_cuda_graph=graph)
        x, inter = s.sample(steps=steps, shape=shape, x_info={"type": "image", "xt": xt}, c_info=c_info, eta=0.0,
                            log_every_t=1)
    return x.clone(), inter


@pytest.mark.parametrize("control", [False, True])
@pytest.mark.parametrize("kind", ["ddim", "dpmpp_2m", "euler_a"])
def test_pipeline_batch_invariant(env, det, kind, control):
    net, inp = env
    x3, inter3 = _sample(net, inp, kind, slice(0, 3), control)
    im3 = net.vae_decode(x3, "image").clone()
    for i in range(3):
        x1, inter1 = _sample(net, inp, kind, slice(i, i + 1), control)
        assert_same(x1[0], x3[i], f"{kind} final latent, sample {i}")
        for key in ("pred_xt", "pred_x0"):
            assert len(inter1[key]) == len(inter3[key])
            for k, (a, b) in enumerate(zip(inter1[key], inter3[key])):
                assert_same(a[0], b[i], f"{kind} {key}[{k}], sample {i}")
        assert_same(net.vae_decode(x1, "image")[0], im3[i], f"{kind} decoded image, sample {i}")
    # a second call (graph replay) and the eager path give the same bits
    assert_same(_sample(net, inp, kind, slice(0, 3), control)[0], x3, f"{kind} second call")
    assert_same(_sample(net, inp, kind, slice(0, 3), control, graph=False)[0], x3, f"{kind} eager vs graph")


def test_seecoder_context_stable(env, det):
    """SeeCoder encodes one reference image per call: the context is the same on graph replay, eagerly, and after
    another image went through the same graph."""
    net, inp = env
    img = inp["img"]
    c1 = net.ctx_encode(img, "image").clone()
    assert_same(net.ctx_encode(img, "image"), c1, "context, graph replay")
    net.ctx_encode(img.flip(3), "image")
    assert_same(net.ctx_encode(img, "image"), c1, "context, replay after another image")
    net.use_cuda_graphs = False
    try:
        assert_same(net.ctx_encode(img, "image"), c1, "context, eager")
    finally:
        net.use_cuda_graphs = True


def test_hed_batch_invariant(det):
    from oracle.hed_oracle import fill_synthetic
    from pfd_b200 import hed
    saved = hed._network
    hed.set_network(fill_synthetic(hed.ControlNetHED().cuda(), seed=0))
    try:
        g = torch.Generator().manual_seed(3)
        x = torch.rand((2, 3, 160, 192), generator=g).cuda()
        both = hed.preprocess_hed(x).clone()
        for i in range(2):
            assert_same(hed.preprocess_hed(x[i:i + 1].contiguous())[0], both[i], f"HED sample {i}")
        assert_same(hed.preprocess_hed(x), both, "HED second call")
    finally:
        hed.set_network(saved)


def test_unet_plan_sms_invariant(env, nv, det):
    net, inp = env
    unet = net.diffuser["image"]
    g = torch.Generator().manual_seed(8)
    x = torch.randn((2, 4, 64, 64), generator=g).cuda().half()
    t = torch.tensor([501, 501], device="cuda")
    c = torch.cat([torch.zeros_like(inp["cond3"][:1]), inp["cond3"][:1]])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    outs = {}
    for plan in (0, 114):
        nv.set_env_option("plan_sms", plan)
        outs[plan] = unet.apply(x, t, c).clone()
    nv.set_env_option("plan_sms", 0)
    assert_same(outs[114], outs[0], f"UNet evaluation planned for 114 vs {sms} SMs")


def test_cross_process_hashes():
    cmd = [sys.executable, os.path.join(ROOT, "tools", "determinism_check.py")]
    lines = []
    for _ in range(2):
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
        got = [l for l in r.stdout.splitlines() if l.startswith("DETERMINISM_RESULT ")]
        assert r.returncode == 0 and got, (r.stdout[-2000:], r.stderr[-2000:])
        lines.append(json.loads(got[-1][len("DETERMINISM_RESULT "):]))
    print(lines[0])
    assert lines[0]["deterministic"] and lines[0] == lines[1], lines


def test_toggle_recaptures_and_stays_close(env):
    import pfd_b200
    from pfd_b200 import DDIMSampler, graphs
    net, inp = env
    was = pfd_b200.is_deterministic()
    s = DDIMSampler(net)
    c_info = {"type": "image", "conditioning": inp["cond3"], "unconditional_conditioning": torch.zeros_like(inp["cond3"]),
              "unconditional_guidance_scale": 2.0, "control": inp["hint"].half()}

    def run():
        x, _ = s.sample(steps=4, shape=[3, 4, 16, 16], x_info={"type": "image", "xt": inp["xt3"]}, c_info=dict(c_info),
                        verbose=False, eta=0.0)
        return net.vae_decode(x, "image").clone(), next(reversed(s._states.values()))

    try:
        pfd_b200.set_deterministic(True)
        gen = graphs.generation()
        im_det, st_det = run()
        assert run()[1] is st_det                                   # same mode: the cached graph is replayed
        pfd_b200.set_deterministic(False)
        assert graphs.generation() > gen and not pfd_b200.is_deterministic()
        im_def, st_def = run()
        assert st_def is not st_det                                 # the switch forced a new capture
        pfd_b200.set_deterministic(True)
        im_det2, st_det2 = run()
        assert st_det2 is not st_det and st_det2 is not st_def
        assert_same(im_det2, im_det, "deterministic images after switching back")
        assert rel_rms(im_def, im_det) < 3e-3
    finally:
        pfd_b200.set_deterministic(was)


def test_two_gpu_split_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29534", os.path.join(ROOT, "tools", "split_check.py"), "--deterministic"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("SPLIT_RESULT ")]
    assert r.returncode == 0 and lines, (r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(lines[-1][len("SPLIT_RESULT "):])
    print(res)
    assert res["deterministic"] and res["exact_equal"]
