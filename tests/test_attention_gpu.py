"""Attention kernels against float64: the flash kernel (both entry points) at every head dim, tile edge and row-max
order with an error bound derived from its arithmetic (attention_ref.py), exact retrieval, padding that must never be
read, output placement in a larger buffer, the row-softmax kernel of the unfused path, and the wrappers' argument
checks.  test_attention_model_cpu.py shows on the CPU that these checks reject subtly wrong variants of the kernel."""
import pytest
import torch

from attention_ref import (HEAD_DIM_CASES, K_BOUND, RETRIEVAL_CASES, ROW_MAX_CASES, TILE_EDGE_CASES, flash_check,
                           flash_inputs, retrieval_inputs, rh, softmax_bound, softmax_ref, ulp16)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


def ceil8(n):
    return (n + 7) // 8 * 8


def packed(q, k, v, B, heads, q_pad=0, k_pad=0, fill=None):
    """Packed layout of native.flash_attn: q [G, Nqp, d], k [G, Nkp, d], vt [G, d, Nkp] on the GPU.  Padding rows /
    columns are zero, or (fill=True) NaN in q and V^T and copies of 4 q in k (keys that would win every row)."""
    G, Nq, d = q.shape
    Nk = k.shape[1]
    Nqp, Nkp = ceil8(Nq) + q_pad, ceil8(Nk) + k_pad
    qp = torch.zeros((G, Nqp, d), dtype=torch.float16)
    kp = torch.zeros((G, Nkp, d), dtype=torch.float16)
    vtp = torch.zeros((G, d, Nkp), dtype=torch.float16)
    if fill:
        qp[:, Nq:] = float("nan")
        kp[:, Nk:] = 4 * q[:, torch.arange(Nk, Nkp) % Nq]
        vtp[:, :, Nk:] = float("nan")
    qp[:, :Nq], kp[:, :Nk], vtp[:, :, :Nk] = q, k, v.transpose(1, 2)
    return qp.cuda(), kp.cuda(), vtp.cuda()


def strided(q, k, v, B, heads, pad=0, fill=None):
    """The UNet self-attention layout (attention.project_heads_fused / project_vt_swapped): q and k are the two head
    sections of one [B, 2*heads, Np, d] buffer, V^T is a [B, heads, d, Nkp] view of a [heads*d, B*Nkp] buffer.
    Padding as in packed(); pad > 0 adds rows to k past its last key so the view does not end at its head."""
    G, Nq, d = q.shape
    Nk = k.shape[1]
    Np = max(ceil8(Nq), ceil8(Nk)) + pad
    Nkp = ceil8(Nk) + pad
    qk = torch.zeros((B, 2 * heads, Np, d), dtype=torch.float16)
    vbuf = torch.zeros((heads * d, B * Nkp), dtype=torch.float16)
    v4 = vbuf.as_strided((B, heads, d, Nkp), (Nkp, d * B * Nkp, B * Nkp, 1))
    if fill:
        qk[:, :heads, Nq:] = float("nan")
        qk[:, heads:, Nk:] = 4 * q.reshape(B, heads, Nq, d)[:, :, torch.arange(Nk, Np) % Nq]
        v4[..., Nk:] = float("nan")
    qk[:, :heads, :Nq] = q.reshape(B, heads, Nq, d)
    qk[:, heads:, :Nk] = k.reshape(B, heads, Nk, d)
    v4[..., :Nk] = v.reshape(B, heads, Nk, d).transpose(2, 3)
    qk, vbuf = qk.cuda(), vbuf.cuda()
    return qk[:, :heads], qk[:, heads:], vbuf.as_strided((B, heads, d, Nkp), (Nkp, d * B * Nkp, B * Nkp, 1))


def run_flash(nv, entry, q, k, v, B, heads, scale, out=None, **layout):
    """One call of an entry point on CPU fp16 inputs; asserts a single launch.  Returns out."""
    G, Nq, d = q.shape
    Nk = k.shape[1]
    if out is None:
        out = torch.full((B, Nq, heads * d), float("nan"), device="cuda", dtype=torch.float16)
    n0 = nv.launch_count()
    if entry == "packed":
        qg, kg, vtg = packed(q, k, v, B, heads, **layout)
        nv.flash_attn(qg, kg, vtg, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale, out=out)
    else:
        qg, kg, vtg = strided(q, k, v, B, heads, **layout)
        nv.flash_attn_strided(qg, kg, vtg, Nq=Nq, Nk=Nk, scale=scale, out=out)
    assert nv.launch_count() == n0 + 1
    torch.cuda.synchronize()
    return out


def per_head(out, B, heads):
    """[B, Nq, heads*d] -> [B*heads, Nq, d]."""
    Bo, Nq, C = out.shape
    return out.reshape(B, Nq, heads, C // heads).permute(0, 2, 1, 3).reshape(B * heads, Nq, C // heads)


ENTRIES = ("packed", "strided")


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", HEAD_DIM_CASES + TILE_EDGE_CASES + ROW_MAX_CASES,
                         ids=lambda c: "B{}h{}q{}k{}d{}-{}".format(*c))
def test_flash_f64(nv, case, entry):
    B, heads, Nq, Nk, d, kind = case
    q, k, v, scale = flash_inputs(*case)
    out = run_flash(nv, entry, q, k, v, B, heads, scale)
    flash_check(per_head(out, B, heads), q.cuda(), k.cuda(), v.cuda(), scale, f"{entry} {case}")


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", RETRIEVAL_CASES, ids=lambda c: "B{}h{}q{}k{}d{}{}".format(*c[:5], "-ghost" * c[5]))
def test_flash_exact_retrieval(nv, case, entry):
    B, heads = case[:2]
    q, k, v, expect = retrieval_inputs(*case)
    out = run_flash(nv, entry, q, k, v, B, heads, 1.0)
    got = per_head(out, B, heads).cpu()
    bad = (got != expect).any(-1)
    assert torch.equal(got, expect), f"{int(bad.sum())} rows differ, first (head, query) {bad.nonzero()[:4].tolist()}"


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("d", (40, 72, 160))
def test_flash_padding_and_output_placement(nv, d, entry):
    """Padding rows of q and k and padding columns of V^T hold NaN or keys that would win every row, and the output is
    a view into a larger NaN buffer (row pitch > heads*d, column offset 8): the result must equal the zero-padding,
    contiguous-output run bit for bit, and nothing outside the view may change."""
    B, heads, Nq, Nk = 2, 3, 130, 77
    q, k, v, scale = flash_inputs(B, heads, Nq, Nk, d, "random", seed=5)
    ref = run_flash(nv, entry, q, k, v, B, heads, scale)
    C = heads * d
    buf = torch.full((B, Nq + 3, C + 40), float("nan"), device="cuda", dtype=torch.float16)
    buf.view(torch.int16)[:, :, ::3] = 0x7E01                       # a second NaN payload
    before = buf.clone()
    view = buf[:, 1:Nq + 1, 8:8 + C]
    pad = dict(k_pad=24, q_pad=16, fill=True) if entry == "packed" else dict(pad=24, fill=True)
    run_flash(nv, entry, q, k, v, B, heads, scale, out=view, **pad)
    assert torch.isfinite(ref.float()).all()
    assert torch.equal(view, ref)
    outside = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    outside[:, 1:Nq + 1, 8:8 + C] = False
    assert torch.equal(buf.view(torch.int16)[outside], before.view(torch.int16)[outside])


# ---------------------------------------------------------------------------------------------- softmax kernel
def softmax_check(out, x, scale, bias=None, mask=None, label=""):
    p, t = softmax_ref(x, scale, bias, mask)
    err = (out.double() - p).abs()
    worst = float((err / softmax_bound(p, t)).max())
    print(f"[softmax f64] {label}: max err/bound {worst:.3f}")
    assert torch.isfinite(out).all() and worst <= 1.0


@pytest.mark.parametrize("cols", (1, 2, 31, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 36864, 50176))
def test_softmax_cols_and_pitch(nv, cols):
    """Row softmax at both sides of the 64 / 128 / 256-thread switch up to the 50176-column limit, in rows padded to
    ld > cols: the canary columns past cols stay untouched."""
    batch, rows, ld = 2, 3, ceil8(cols) + 8
    g = torch.Generator().manual_seed(cols)
    x = (torch.randn((batch, rows, cols), generator=g) * 6).half().cuda()
    buf = torch.full((batch, rows, ld), 7.0, device="cuda", dtype=torch.float16)
    buf[..., :cols] = x
    before = buf.clone()
    n0 = nv.launch_count()
    nv.softmax_(buf[..., :cols], 0.125)
    assert nv.launch_count() == n0 + 1
    torch.cuda.synchronize()
    assert torch.equal(buf[..., cols:], before[..., cols:])
    softmax_check(buf[..., :cols], x, 0.125, label=f"cols {cols} ld {ld}")


@pytest.mark.parametrize("swin_mask", (False, True))
def test_softmax_bias_mask_mapping(nv, swin_mask):
    """batch = 2 * nheads * nwin rows of heads: bias row b % nheads, mask row (b / nheads) % nwin, with distinct values
    per head and per window; swin_mask uses the 0 / -100 shift mask."""
    nheads, nwin, rows, cols = 3, 4, 144, 144
    batch = 2 * nheads * nwin
    g = torch.Generator().manual_seed(11)
    x = (torch.randn((batch, rows, cols), generator=g) * 4).half().cuda()
    bias = (torch.randn((nheads, rows, cols), generator=g) + torch.arange(nheads)[:, None, None]).half().cuda()
    if swin_mask:
        mask = torch.where(torch.rand((nwin, rows, cols), generator=g) < 0.4, -100.0, 0.0).half().cuda()
    else:
        mask = (torch.randn((nwin, rows, cols), generator=g) - 2 * torch.arange(nwin)[:, None, None]).half().cuda()
    s = x.clone()
    nv.softmax_(s, 0.17, bias=bias, nheads=nheads, mask=mask, nwin=nwin)
    torch.cuda.synchronize()
    b = torch.arange(batch, device="cuda")
    softmax_check(s, x, 0.17, bias[b % nheads], mask[(b // nheads) % nwin], f"bias/mask swin={swin_mask}")


# ---------------------------------------------------------------------------------------------- unfused attend
def unfused_ref_bound(q, k, vt, scale, Nk, bias=None, mask=None):
    """Float64 attention with the reference's fp16 rounding points (scores, scaled scores (+ bias, + mask),
    probabilities) and a bound on the kernels' deviation from it.

    Given the same fp16 scores, the softmax kernel reproduces the rounded logits bit for bit, so the logits can differ
    only where the score GEMM's fp32 accumulation error (d 2^-24 sum |q k|) straddles an fp16 rounding boundary of
    S: both roundings are evaluated there.  A probability can round the other way only where the softmax kernel's
    fp32 error (and such a logit change) reaches its fp16 rounding boundary: both roundings again.  Then the fp32 PV
    accumulation and, as in the flash bound, one ulp of output rounding."""
    Sx = q.double() @ k[:, :Nk].double().transpose(1, 2)
    eS = K_BOUND * q.shape[-1] * 2.0 ** -24 * (q.double().abs() @ k[:, :Nk].double().abs().transpose(1, 2))
    p, t = softmax_ref(rh(Sx), scale, bias, mask)
    dt = torch.maximum((softmax_ref(rh(Sx - eS), scale, bias, mask)[1] - t).abs(),
                       (softmax_ref(rh(Sx + eS), scale, bias, mask)[1] - t).abs())
    # relative change of p_j under logit changes dt: exp(dt_j + sum_i p_i dt_i) - 1, plus the kernel's fp32 error
    rel = torch.expm1(dt + (p * dt).sum(-1, keepdim=True)) + (softmax_bound(p, t) - ulp16(p)) / p.clamp_min(1e-300)
    dp = p * rel
    P = rh(p)
    dP = torch.maximum((rh(p + dp) - P).abs(), (rh(p - dp) - P).abs())
    V = vt[:, :, :Nk].double().transpose(1, 2)
    O = P @ V
    E = K_BOUND * (dP @ V.abs() + Nk * 2.0 ** -24 * (P @ V.abs()))
    return O, E + ulp16(O.abs() + E)


@pytest.mark.parametrize("d,N,bias_mask", [(32, 144, True), (256, 77, False)])
def test_attend_unfused(nv, d, N, bias_mask):
    """Swin window attention (nwin windows x heads, N = 144, d = 32, relative-position bias and -100 shift mask)
    through attention.attend, and d = 256, which falls back from flash to the GEMM -> softmax -> GEMM path."""
    from pfd_b200 import attention as att
    B, heads, nwin = (2 * 4, 3, 4) if bias_mask else (1, 2, 1)
    G, Np = B * heads, ceil8(N)
    g = torch.Generator().manual_seed(d)
    q = torch.zeros((G, Np, d), dtype=torch.float16)
    k = torch.zeros((G, Np, d), dtype=torch.float16)
    vt = torch.zeros((G, d, Np), dtype=torch.float16)
    q[:, :N] = torch.randn((G, N, d), generator=g).half()
    k[:, :N] = torch.randn((G, N, d), generator=g).half()
    vt[:, :, :N] = torch.randn((G, d, N), generator=g).half()
    q, k, vt = q.cuda(), k.cuda(), vt.cuda()
    bias = mask = None
    if bias_mask:
        bias = (torch.randn((heads, N, N), generator=g) * 2).half().cuda()
        mask = torch.where(torch.rand((nwin, N, N), generator=g) < 0.4, -100.0, 0.0).half().cuda()
    scale = d ** -0.5
    out = att.attend(q, k, vt, B=B, heads=heads, Nq=N, Nk=N, scale=scale, bias=bias, mask=mask, nwin=nwin)
    torch.cuda.synchronize()
    b = torch.arange(G, device="cuda")
    O, bound = unfused_ref_bound(q[:, :N], k, vt, scale, N, None if bias is None else bias[b % heads],
                                 None if mask is None else mask[(b // heads) % nwin])
    got = per_head(out, B, heads).double()
    worst = float(((got - O).abs() / bound).max())
    rel = float((bound / O.abs().clamp_min(2.0 ** -14)).median())
    print(f"[attend unfused f64] d={d} N={N} bias/mask={bias_mask}: max err/bound {worst:.3f}, "
          f"median bound/|O| {rel:.2e}")
    assert torch.isfinite(got).all() and worst <= 1.0


# ---------------------------------------------------------------------------------------------- wrapper checks
class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"malformed call reached the library ({name})")


def _malformed_calls(nv):
    h = torch.float16
    z = lambda *s: torch.zeros(s, device="cuda", dtype=h)
    B, H, N, d = 2, 2, 16, 16
    q, k, vt, out = z(B * H, N, d), z(B * H, N, d), z(B * H, d, N), z(B, N, H * d)
    fa = lambda q=q, k=k, vt=vt, out=out, Nq=N, Nk=N: nv.flash_attn(q, k, vt, B=B, heads=H, Nq=Nq, Nk=Nk,
                                                                     scale=0.25, out=out)
    qk = z(B, 2 * H, N, d)
    vt4 = z(B, H, d, N)
    fs = lambda q=qk[:, :H], k=qk[:, H:], vt=vt4, out=out, Nq=N, Nk=N: nv.flash_attn_strided(
        q, k, vt, Nq=Nq, Nk=Nk, scale=0.25, out=out)
    s = z(4, 8, 32)
    sm = lambda s=s, **kw: nv.softmax_(s, 0.5, **kw)
    return {
        "flash Nq > q rows": lambda: fa(Nq=N + 1),
        "flash Nq = 0": lambda: fa(Nq=0),
        "flash Nk > k rows": lambda: fa(k=z(B * H, N - 8, d)),
        "flash Nk > vt cols": lambda: fa(vt=z(B * H, d, N - 8)),
        "flash k head dim": lambda: fa(k=z(B * H, N, d + 8)),
        "flash vt rows != d": lambda: fa(vt=z(B * H, d + 8, N)),
        "flash q heads": lambda: fa(q=z(B * H + 1, N, d)),
        "flash q not contiguous": lambda: fa(q=z(B * H, N, 2 * d)[..., :d]),
        "flash q inner stride": lambda: fa(q=z(B * H, N, 2 * d)[..., ::2]),
        "flash vt inner stride": lambda: fa(vt=z(B * H, d, 2 * N)[..., ::2]),
        "flash out inner stride": lambda: fa(out=z(B, N, 2 * H * d)[..., ::2]),
        "flash out too narrow": lambda: fa(out=z(B, N, H * d - 8)),
        "flash out too few rows": lambda: fa(out=z(B, N - 1, H * d)),
        "flash out odd row stride": lambda: fa(out=z(B, N, H * d + 1)[..., :H * d]),
        "flash out odd batch stride": lambda: fa(out=z(B * N * H * d + 8).as_strided((B, N, H * d),
                                                                                      (N * H * d + 1, H * d, 1))),
        "flash out misaligned": lambda: fa(out=z(B, N, H * d + 8)[..., 1:H * d + 1]),
        "flash out dtype": lambda: fa(out=out.float()),
        "strided Nk > k rows": lambda: fs(k=qk[:, H:, :N - 8]),
        "strided Nk > vt cols": lambda: fs(vt=vt4[..., :N - 8]),
        "strided Nq > q rows": lambda: fs(Nq=N + 8),
        "strided k head dim": lambda: fs(k=z(B, H, N, d + 8)),
        "strided vt rows != d": lambda: fs(vt=z(B, H, d + 8, N)),
        "strided k heads": lambda: fs(k=qk[:, H + 1:]),
        "strided k inner stride": lambda: fs(k=z(B, H, N, 2 * d)[..., ::2]),
        "strided vt inner stride": lambda: fs(vt=z(B, H, d, 2 * N)[..., ::2]),
        "strided out misaligned": lambda: fs(out=z(B, N, H * d + 8)[..., 1:H * d + 1]),
        "softmax inner stride": lambda: sm(s=z(4, 8, 64)[..., ::2]),
        "softmax batch stride": lambda: sm(s=z(4, 16, 32)[:, :8]),
        "softmax row pitch < cols": lambda: sm(s=z(4 * 8 * 32).as_strided((4, 8, 32), (8 * 16, 16, 1))),
        "softmax bias shape": lambda: sm(bias=z(2, 8, 32), nheads=4),
        "softmax bias not contiguous": lambda: sm(bias=z(2, 8, 64)[..., :32], nheads=2),
        "softmax mask shape": lambda: sm(mask=z(2, 8, 16), nwin=2),
        "softmax mask nwin": lambda: sm(mask=z(3, 8, 32), nwin=2),
    }


def test_wrapper_argument_checks(nv, monkeypatch):
    """Each malformed call raises on the host before the library is called (the library is replaced by an object that
    fails any use), and the launch counter does not move."""
    lib = nv.load()
    calls = _malformed_calls(nv)
    n0 = lib.pfd_launch_count()
    monkeypatch.setattr(nv, "load", lambda: _NoLibrary())
    failures = []
    for name, call in calls.items():
        try:
            call()
            failures.append(f"{name}: accepted")
        except ValueError:
            pass
        except RuntimeError as e:                   # the wrappers' dtype / device check
            if "expected a CUDA fp16 tensor" not in str(e):
                failures.append(f"{name}: {e}")
        except AssertionError as e:                 # reached the library stub
            failures.append(f"{name}: {e}")
    monkeypatch.undo()
    assert lib.pfd_launch_count() == n0
    assert not failures, failures
