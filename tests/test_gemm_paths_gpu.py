"""Exact-arithmetic tests of the GEMM paths the network runs outside the common 3x3 / 64-channel case: narrow-channel
3x3 convs (a_c % 64 != 0, the ControlNet hint stem), stride 2 on odd and non-square rasters with tap_off 0 and 1 (the
VAE encoder's downsample), alpha != 1, and split-K with its finish kernel under every epilogue feature and output
addressing, ragged N and batched B.

Operands are small integers (B scaled by a power of two for the SiLU / GELU cases), so every product and partial sum
is exactly representable in fp32 and the accumulator is the same in any K order, split or not.  The fractional bits
sit in bias, row add and residual, so the epilogue's rounding points decide the last bit.  The reference is an fp64
model of the documented contract

    y = fp16(act(acc * alpha + bias + rowadd)),   out = fp16(y + residual)

compared bit for bit for ACT_NONE and ReLU.  SiLU and GELU may differ by one fp16 ulp of y (and one of out when a
residual is added): their fp32 approximations (__expf, fast_erf to 1.5e-7) can move a value across a rounding boundary.
Every plan of a case (each planning SM count, each forced N tile width, deterministic mode) must give the same bits,
and the number of kernels each plan launched (1 = one GEMM, 2 = GEMM + split-K finish) is checked against the
planner's expected choice for 132-, 114-, 66- and 16-SM plans."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PLANS = (0, 114, 66, 16)            # plan_sms values; 0 = the device's SM count
WIDTHS = (64, 128, 160, 192, 256)   # forced N tile widths (never split K)
SPLIT_ALL = {132: 2, 114: 2, 66: 2, 16: 2}
SPLIT_BUT_16 = {132: 2, 114: 2, 66: 2, 16: 1}


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


# ----------------------------------------------------------------------------------------------- operands
def ints(shape, seed, scale=1.0):
    """fp16 integers in {-2, ..., 2}, times `scale` (a power of two)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-2, 3, shape, generator=g).double() * scale).to("cuda", torch.float16)


def fracs(shape, seed, mag, step):
    """fp16 multiples of `step` (a power of two) in [-mag, mag]; fp16 keeps them multiples of step."""
    g = torch.Generator().manual_seed(seed)
    n = int(mag / step)
    return (torch.randint(-n, n + 1, shape, generator=g).double() * step).to("cuda", torch.float16)


def ulp16(x):
    """Spacing of the fp16 values at |x| (float64 in, float64 out)."""
    _, e = torch.frexp(x.double())
    return torch.pow(2.0, (torch.clamp(e - 1, min=-14) - 10).double())


def half_rn(x):
    """float64 -> fp16 rounded once, to nearest even (a plain .half() goes through float32 and can round twice)."""
    q = ulp16(x)
    return (torch.round(x / q) * q).to(torch.float16)


ACTS = {"none": 0, "silu": 1, "gelu": 2, "relu": 3}


def act64(v, act):
    if act == "silu":
        return v * torch.sigmoid(v)
    if act == "gelu":
        return F.gelu(v)
    if act == "relu":
        return v.clamp(min=0)
    return v


# ----------------------------------------------------------------------------------------------- output layouts
def layout(kind, NB, H, W, N):
    """(buffer shape, so, ndiv, cdiv, view of a buffer as the canonical [NB, H, W, N])."""
    if kind == "nhwc":
        return (NB, H, W, N), (H * W * N, 0, W * N, N, 0, 1), 1, 0, lambda t: t
    if kind == "nchw":                 # element-strided columns: scalar stores
        return (NB, N, H, W), (N * H * W, 0, W, 1, 0, H * W), 1, 0, lambda t: t.permute(0, 2, 3, 1)
    if kind.startswith("heads_t"):     # [NB, heads, d, H, W] (V^T-like): head split and element-strided columns
        d = int(kind[7:])
        return ((NB, N // d, d, H, W), (N * H * W, 0, W, 1, d * H * W, H * W), 1, d,
                lambda t: t.permute(0, 3, 4, 1, 2).reshape(NB, H, W, N))
    if kind.startswith("heads"):       # [NB, heads, H, W, d]
        d = int(kind[5:])
        return ((NB, N // d, H, W, d), (N * H * W, 0, W * d, d, H * W * d, 1), 1, d,
                lambda t: t.permute(0, 2, 3, 1, 4).reshape(NB, H, W, N))
    if kind.startswith("ndiv"):        # image n -> [n / h, y, x, n % h, :] (the attention P.V output with h = heads)
        h = int(kind[4:])
        return ((NB // h, H, W, h, N), (H * W * h * N, N, W * h * N, h * N, 0, 1), h, 0,
                lambda t: t.permute(0, 3, 1, 2, 4).reshape(NB, H, W, N))
    raise ValueError(kind)


# ----------------------------------------------------------------------------------------------- cases
def conv(NB, H, W, C, N, stride=1, tap_off=0, **kw):
    return dict(op="conv", NB=NB, H=H, W=W, C=C, N=N, stride=stride, tap_off=tap_off, **kw)


def linear(M, K, N, **kw):
    return dict(op="linear", M=M, K=K, N=N, **kw)


def bmm(B, M, K, N, **kw):
    return dict(op="bmm", B=B, M=M, K=K, N=N, **kw)


CASES = {}
# ControlNet hint stem at a 512x512 hint (3x3, bias, SiLU; channel counts that leave part of each 64-wide K block to
# the TMA zero fill), plus the same convs with a residual and no activation for bit equality, and C = 8 / 40
for H, C, N, s in ((512, 16, 16, 1), (512, 16, 32, 2), (256, 32, 32, 1), (256, 32, 96, 2), (128, 96, 96, 1),
                   (128, 96, 256, 2), (80, 8, 48, 1), (72, 40, 88, 2)):
    CASES[f"stem_{H}_{C}to{N}_s{s}_silu"] = conv(1, H, H, C, N, s, act="silu", bias=True, launches=1)
    CASES[f"stem_{H}_{C}to{N}_s{s}_res"] = conv(1, H, H, C, N, s, act="none", bias=True, residual=True, launches=1)
# stride 2 with tap_off = 1 (F.pad(x, (0, 1, 0, 1)) + padding 0, the VAE encoder's downsample) and tap_off = 0
CASES["vae_down_512"] = conv(1, 512, 512, 128, 128, 2, 1, act="none", bias=True, launches=1)
for H, W in ((33, 47), (9, 5), (3, 3), (1, 1)):
    for t in (0, 1):
        if (H - 1 - t) // 2 + 1 > 0 and (W - 1 - t) // 2 + 1 > 0:
            CASES[f"s2_{H}x{W}_tap{t}"] = conv(2, H, W, 64, 136, 2, t, act="none", bias=True, residual=True,
                                               launches=1)
# alpha != 1 on a Linear with bias and residual: short K (staged epilogue) and K = 5120 (split-K)
for a in (0.5, 0.125):
    CASES[f"alpha{a}_staged"] = linear(1000, 320, 328, act="none", alpha=a, bias=True, residual=True, launches=1)
    CASES[f"alpha{a}_splitk"] = linear(256, 5120, 640, act="none", alpha=a, bias=True, residual=True,
                                       launches=SPLIT_ALL)
# split-K epilogue matrix: 3x3 at 8x8, C = 1280 (K = 11520) on two images, ragged N (the finish kernel's N tile falls
# back to 128)
SPLITK_FEATURES = {
    "bias_res": dict(act="none", bias=True, residual=True),
    "rowadd_silu_res": dict(act="silu", bias=True, rowadd=True, residual=True),
    "gelu_res_inplace": dict(act="gelu", bias=True, residual=True, inplace=True),
    "relu_res_nchw": dict(act="relu", bias=True, residual=True, out="nchw"),
    "rowadd_relu_res_ndiv2": dict(act="relu", rowadd=True, residual=True, out="ndiv2"),
    "bias_res_heads": dict(act="none", bias=True, residual=True, out="heads"),
    "rowadd_res_heads_t": dict(act="none", rowadd=True, residual=True, out="heads_t"),
    "bias_res_heads4": dict(act="none", bias=True, residual=True, out="heads4"),   # 4-wide heads: scalar stores
}
for N, d in ((200, 40), (328, 8)):
    for name, f in SPLITK_FEATURES.items():
        f = dict(f)
        if f.get("out") in ("heads", "heads_t"):
            f["out"] += str(d)
        CASES[f"splitk_{name}_n{N}"] = conv(2, 8, 8, 1280, N, launches=SPLIT_ALL, **f)
CASES["splitk_resblock_out_1280"] = conv(8, 8, 8, 1280, 1280, act="none", bias=True, residual=True,
                                         launches=SPLIT_BUT_16)
CASES["splitk_c2560_rowadd_silu_res"] = conv(2, 8, 8, 2560, 640, act="silu", bias=True, rowadd=True, residual=True,
                                             launches=SPLIT_ALL)
CASES["splitk_linear_m77_res_inplace"] = linear(77, 5120, 200, act="none", bias=True, residual=True, inplace=True,
                                                launches=SPLIT_ALL)
CASES["splitk_linear_m256_gelu_res"] = linear(256, 5120, 328, act="gelu", bias=True, residual=True,
                                              launches=SPLIT_ALL)
# split-K with a batched B operand: the VAE mid-attention P.V at batch 1 (all 4096 query rows, and a ragged chunk),
# and the unfused attention P.V with its [B, Nq, heads*d] output (ndiv = heads)
CASES["splitk_vae_pv_4096"] = bmm(1, 4096, 4096, 512, act="none", launches={132: 2, 114: 1, 66: 1, 16: 1})
CASES["splitk_vae_pv_1000"] = bmm(1, 1000, 4096, 512, act="none", launches=SPLIT_BUT_16)
CASES["splitk_attn_pv_ndiv8"] = bmm(8, 200, 2048, 40, act="none", out="ndiv8", launches=SPLIT_BUT_16)


def build(nv, spec):
    """(run(bn_force) -> output in canonical layout, fp64 accumulator, epilogue tensors) of one case."""
    act = spec["act"]
    op, N = spec["op"], spec["N"]
    if op == "conv":
        NB, H, W, C, s, t = spec["NB"], spec["H"], spec["W"], spec["C"], spec["stride"], spec["tap_off"]
        Ho, Wo, K = (H - 1 - t) // s + 1, (W - 1 - t) // s + 1, 9 * C
    elif op == "linear":
        NB, Ho, Wo, K = 1, 1, spec["M"], spec["K"]
    else:
        NB, Ho, Wo, K = spec["B"], 1, spec["M"], spec["K"]
    exact = act in ("none", "relu")
    # SiLU / GELU need pre-activations of order 1: scale B so the accumulator's spread is about 1
    bscale = 1.0 if exact else 2.0 ** -round(math.log2(2 * math.sqrt(K)))
    seed = sum(map(ord, repr(sorted(spec.items()))))
    if op == "conv":
        x = ints((NB, H, W, C), seed)
        w4 = ints((N, C, 3, 3), seed + 1, bscale)
        wp = w4.permute(0, 2, 3, 1).reshape(N, K).contiguous()
        xr = x.double().permute(0, 3, 1, 2)
        if t:
            acc = F.conv2d(F.pad(xr, (0, 1, 0, 1)), w4.double(), stride=s)
        else:
            acc = F.conv2d(xr, w4.double(), stride=s, padding=1)
        acc = acc.permute(0, 2, 3, 1)
        segs = [(x, 9, C, (x.stride(2), x.stride(1), x.stride(0)))]
        geo = dict(in_w=W, in_h=H, stride=s, W=Wo, H=Ho, NB=NB, w=wp, N=N, K=K, tap_off=t)
    elif op == "linear":
        x, w = ints((Wo, K), seed), ints((N, K), seed + 1, bscale)
        acc = (x.double() @ w.double().t()).reshape(1, 1, Wo, N)
        segs = [(x, 1, K, (K, K * Wo, K * Wo))]
        geo = dict(in_w=Wo, in_h=1, stride=1, W=Wo, H=1, NB=1, w=w, N=N, K=K)
    else:
        a, b = ints((NB, Wo, K), seed), ints((NB, N, K), seed + 1, bscale)
        acc = torch.bmm(a.double(), b.double().transpose(1, 2)).reshape(NB, 1, Wo, N)
        segs = [(a, 1, K, (K, K * Wo, K * Wo))]
        geo = dict(in_w=Wo, in_h=1, stride=1, W=Wo, H=1, NB=NB, w=b, N=N, K=K, b_batch_stride=N * K)
    assert (acc / bscale).abs().max().item() < 2048, "accumulator outside the exactly summed range"

    shape, so, ndiv, cdiv, canon = layout(spec.get("out", "nhwc"), NB, Ho, Wo, N)
    bias = fracs((N,), seed + 2, 512, 1 / 8) if exact else fracs((N,), seed + 2, 2, 1 / 64)
    rowadd = None
    if spec.get("rowadd"):
        big = fracs((NB, N + 24), seed + 3, 256, 1 / 8) if exact else fracs((NB, N + 24), seed + 3, 1, 1 / 64)
        rowadd = big[:, :N]                                 # row pitch N + 24 > N
    residual = fracs(shape, seed + 4, 512, 1 / 8) if spec.get("residual") else None
    ep = dict(alpha=spec.get("alpha", 1.0), act=act, bias=bias if spec.get("bias") else None, rowadd=rowadd,
              residual=None if residual is None else canon(residual))

    def run(bn):
        if spec.get("inplace"):
            out = residual.clone()
            res = out
        else:
            out = torch.empty(shape, device="cuda", dtype=torch.float16)
            res = residual
        nv.gemm_raw(segs, **geo, alpha=ep["alpha"], act=ACTS[act], bias=ep["bias"], rowadd=rowadd, residual=res,
                    out=out, so=so, ndiv=ndiv, cdiv=cdiv, bn_force=bn)
        return canon(out)
    return run, acc, ep


def model(acc, ep):
    """fp64 model of the contract: (out, y, out rounded once or None without a residual, pre-activation v)."""
    v = acc * ep["alpha"]
    if ep["bias"] is not None:
        v = v + ep["bias"].double()
    if ep["rowadd"] is not None:
        v = v + ep["rowadd"].double()[:, None, None, :]
    y = half_rn(act64(v, ep["act"]))
    if ep["residual"] is None:
        return y, y, None, v
    r = ep["residual"].double()
    return half_rn(y.double() + r), y, half_rn(act64(v, ep["act"]) + r), v


def bits(t):
    return t.contiguous().view(torch.int16)


def run_plans(nv, run, launches):
    """Output of every plan of a case, keyed by plan; asserts the kernels each plan launched."""
    import pfd_b200
    dev = torch.cuda.get_device_properties(0).multi_processor_count
    was = pfd_b200.is_deterministic()
    outs = {}

    def launch(key, bn, want):
        n0 = nv.launch_count()
        o = run(bn).clone()
        got = nv.launch_count() - n0
        if want is not None:
            assert got == want, f"{key}: {got} kernel launches, expected {want}"
        outs[key] = o

    try:
        pfd_b200.set_deterministic(False)
        for plan in PLANS:
            nv.set_env_option("plan_sms", plan)
            sms = min(plan or dev, dev)
            launch(f"plan_sms={sms}", 0, launches if isinstance(launches, int) else launches.get(sms))
        nv.set_env_option("plan_sms", 0)
        for bn in WIDTHS:
            launch(f"bn_force={bn}", bn, 1)
        pfd_b200.set_deterministic(True)
        launch("deterministic", 0, 1)
    finally:
        nv.set_env_option("plan_sms", 0)
        pfd_b200.set_deterministic(was)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("name", list(CASES))
def test_gemm_path_exact(nv, name):
    spec = CASES[name]
    run, acc, ep = build(nv, spec)
    ref, y, once, v = model(acc, ep)
    if once is not None:
        # the case can tell the two rounding orders apart
        assert not torch.equal(ref, once), "no element where rounding y first changes the result"
    outs = run_plans(nv, run, spec["launches"])
    first_key, first = next(iter(outs.items()))
    for key, o in outs.items():
        assert torch.equal(bits(o), bits(first)), \
            f"{key} vs {first_key}: {(bits(o) != bits(first)).sum().item()} elements differ"
    out = first.double()
    if spec["act"] in ("none", "relu"):
        bad = out != ref.double()
        assert not bad.any(), (f"{bad.sum().item()}/{bad.numel()} elements differ from the fp64 model, e.g. "
                               f"{out[bad][:4].tolist()} vs {ref.double()[bad][:4].tolist()}"
                               + ("" if once is None else f" (rounded once: {once.double()[bad][:4].tolist()})"))
    else:
        # one ulp of y, plus the fp32 approximation's error where it exceeds that ulp (GELU's 1 + erf cancels near
        # v << 0, where y is far smaller than fast_erf's 1.5e-7 absolute error times v / 2)
        tol = ulp16(y.double()) + (2e-7 * v.abs() if spec["act"] == "gelu" else 2.0 ** -20 * y.double().abs())
        if ep["residual"] is not None:
            tol = tol + ulp16(torch.maximum(out.abs(), ref.double().abs()))
        err = (out - ref.double()).abs()
        bad = err > tol
        assert not bad.any(), f"{bad.sum().item()}/{bad.numel()} elements off by more than one ulp, max {err.max().item():.3g}"
