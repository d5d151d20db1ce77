"""GPU parity tests of the C-ABI kernels against plain torch fp32 math on the same fp16 inputs.

Every call goes through ctypes -> libpfd_b200.so (pfd_b200/native.py); torch is only the checker.
Tolerances: outputs are fp16, accumulation fp32 -> |err| <= 2^-9 * |ref| + small abs term.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from attention_ref import flash_check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to("cuda", torch.float16)


def close(out, ref, rtol=4e-3, atol=4e-3):
    out = out.float()
    ref = ref.float()
    err = (out - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} mismatches, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 320, 320), (4096, 320, 320), (1000, 1280, 768),
                                   (77, 640, 1280), (512, 24, 40), (300, 2560, 320), (8, 1280, 1280),
                                   (512, 1280, 5120), (100, 640, 4096)])                 # last two: split-K path
def test_linear(nv, M, N, K):
    x = rnd(M, K, scale=1.0)
    w = rnd(N, K, scale=K ** -0.5, seed=1)
    b = rnd(N, seed=2)
    out = nv.linear(x, w, b)
    torch.cuda.synchronize()
    close(out, x.float() @ w.float().t() + b.float())


@pytest.mark.parametrize("act", ["silu", "gelu", "relu"])
def test_linear_act_residual(nv, act):
    M, N, K = 640, 384, 192
    x, w, b, r = rnd(M, K), rnd(N, K, scale=K ** -0.5, seed=1), rnd(N, seed=2), rnd(M, N, seed=3)
    code = {"silu": nv.ACT_SILU, "gelu": nv.ACT_GELU, "relu": nv.ACT_RELU}[act]
    out = nv.linear(x, w, b, act=code, residual=r)
    torch.cuda.synchronize()
    y = x.float() @ w.float().t() + b.float()
    y = {"silu": F.silu, "gelu": F.gelu, "relu": F.relu}[act](y) + r.float()
    close(out, y)


def test_linear_two_segments(nv):
    M, N, K1, K2 = 512, 320, 640, 320
    x1, x2 = rnd(M, K1), rnd(M, K2, seed=5)
    w = rnd(N, K1 + K2, scale=(K1 + K2) ** -0.5, seed=1)
    out = nv.linear(x1, w, None, x2=x2)
    torch.cuda.synchronize()
    close(out, torch.cat([x1, x2], 1).float() @ w.float().t())


@pytest.mark.parametrize("case", ["linear_res", "linear_narrow", "linear_ragged", "linear_slice", "conv_res", "conv_small",
                                  "conv_rowadd_silu", "conv_stride2", "bmm"])
def test_gemm_epilogue_rasters(nv, case):
    """The GEMM epilogue for every raster tiling: 128x1x1 rows (Linear), 8x8x2 / 16x8 / 32x4 pixel tiles (convs),
    ragged rows / columns, N not a multiple of the tile, an output that is a column slice of a wider tensor (the
    columns outside the slice stay untouched), per-image row add + activation, and batched B.  Against torch fp32,
    and a second launch must reproduce the bits."""
    def run():
        if case == "linear_res":
            x, w, b, r = rnd(4096, 320), rnd(320, 320, scale=320 ** -0.5, seed=1), rnd(320, seed=2), rnd(4096, 320, seed=3)
            return nv.linear(x, w, b, residual=r), x.float() @ w.float().t() + b.float() + r.float()
        if case == "linear_narrow":
            x, w, b = rnd(512, 40), rnd(24, 40, scale=40 ** -0.5, seed=1), rnd(24, seed=2)
            return nv.linear(x, w, b), x.float() @ w.float().t() + b.float()
        if case == "linear_ragged":
            x, w, r = rnd(1000, 768), rnd(1288, 768, scale=768 ** -0.5, seed=1), rnd(1000, 1288, seed=3)
            return nv.linear(x, w, None, residual=r), x.float() @ w.float().t() + r.float()
        if case == "linear_slice":
            x, w, b = rnd(300, 192), rnd(320, 192, scale=192 ** -0.5, seed=1), rnd(320, seed=2)
            big = torch.full((300, 1024), 7.0, device="cuda", dtype=torch.float16)
            out = nv.linear(x, w, b, out=big[:, 128:448])
            assert (big[:, :128] == 7).all() and (big[:, 448:] == 7).all()
            return out.contiguous(), x.float() @ w.float().t() + b.float()
        if case in ("conv_res", "conv_small", "conv_rowadd_silu", "conv_stride2"):
            NB, H, W, C, N = {"conv_res": (2, 64, 64, 320, 320), "conv_small": (3, 8, 8, 128, 192),
                              "conv_rowadd_silu": (2, 24, 24, 64, 160), "conv_stride2": (2, 32, 32, 64, 128)}[case]
            x = rnd(NB, H, W, C)
            w4 = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
            b = rnd(N, seed=2)
            wp = w4.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
            xr = x.float().permute(0, 3, 1, 2)
            if case == "conv_stride2":
                out = nv.conv3x3(x, wp, b, stride=2)
                ref = F.conv2d(xr, w4.float(), b.float(), stride=2, padding=1)
            elif case == "conv_rowadd_silu":
                ra = rnd(NB, N, seed=5)
                out = nv.conv3x3(x, wp, b, rowadd=ra, act=nv.ACT_SILU)
                ref = F.silu(F.conv2d(xr, w4.float(), b.float(), padding=1) + ra.float()[:, :, None, None])
            else:
                r = rnd(NB, H, W, N, seed=3)
                out = nv.conv3x3(x, wp, b, residual=r)
                ref = F.conv2d(xr, w4.float(), b.float(), padding=1) + r.float().permute(0, 3, 1, 2)
            return out, ref.permute(0, 2, 3, 1)
        q, k = rnd(6, 200, 64), rnd(6, 136, 64, seed=1)
        s_ = torch.empty((6, 200, 136), device="cuda", dtype=torch.float16)
        nv.gemm_raw([(q, 1, 64, (64, 64 * 200, 64 * 200))], in_w=200, in_h=1, stride=1, W=200, H=1, NB=6, w=k, N=136, K=64,
                    b_batch_stride=136 * 64, out=s_, so=(200 * 136, 0, 0, 136, 0, 1))
        return s_, torch.bmm(q.float(), k.float().transpose(1, 2))
    out0, ref = run()
    out0 = out0.clone()
    out1, _ = run()
    torch.cuda.synchronize()
    close(out0, ref)
    assert torch.equal(out0, out1), f"two launches differ: max |d| = {(out0.float() - out1.float()).abs().max().item()}"


@pytest.mark.parametrize("case", ["conv_res_2tiles", "conv_many_waves", "conv_wide_rowadd_silu", "linear_odd_ragged",
                                  "conv_stride2", "conv_tiny", "conv_skip_segments", "conv_l1", "conv_l2_single_wave",
                                  "conv_l0_res", "linear_bigk_res", "conv_ragged_rowadd_silu"])
def test_gemm_conv_tilings(nv, case):
    """Long-K convs and Linears against torch fp32: one / many tiles per CTA of the persistent kernel (pipeline phases
    across tiles), N tiles 256 / 160 / 128, an odd number of 128-row tiles, N not a multiple of the tile, stride 2,
    per-image row add + SiLU, residual, extra 1x1 K segments.  The UNet's batch-8 level convs (a partially filled last
    wave, or a single wave), a K = 5120 Linear with bias + residual, and 7 images with N = 328 (ragged rows and
    columns)."""
    def run():
        if case == "linear_odd_ragged":
            x, w, r = rnd(640, 1024), rnd(1288, 1024, scale=1024 ** -0.5, seed=1), rnd(640, 1288, seed=3)
            return nv.linear(x, w, None, residual=r), x.float() @ w.float().t() + r.float()
        if case == "linear_bigk_res":
            x, w, b, r = rnd(2048, 5120), rnd(1280, 5120, scale=5120 ** -0.5, seed=1), rnd(1280, seed=2), rnd(2048, 1280, seed=3)
            return nv.linear(x, w, b, residual=r), x.float() @ w.float().t() + b.float() + r.float()
        NB, H, W, C, N = {"conv_res_2tiles": (2, 64, 64, 320, 320), "conv_many_waves": (8, 64, 64, 128, 320),
                          "conv_wide_rowadd_silu": (2, 32, 32, 128, 1280), "conv_stride2": (4, 32, 32, 128, 256),
                          "conv_tiny": (3, 8, 8, 128, 128), "conv_skip_segments": (2, 32, 32, 64, 160),
                          "conv_l1": (8, 32, 32, 640, 640), "conv_l2_single_wave": (8, 16, 16, 640, 1280),
                          "conv_l0_res": (8, 64, 64, 320, 320), "conv_ragged_rowadd_silu": (7, 24, 24, 192, 328)}[case]
        x = rnd(NB, H, W, C)
        w4 = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
        b = rnd(N, seed=2)
        wp = w4.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
        xr = x.float().permute(0, 3, 1, 2)
        if case == "conv_stride2":
            out = nv.conv3x3(x, wp, b, stride=2)
            ref = F.conv2d(xr, w4.float(), b.float(), stride=2, padding=1)
        elif case in ("conv_l1", "conv_l2_single_wave"):
            out = nv.conv3x3(x, wp, b)
            ref = F.conv2d(xr, w4.float(), b.float(), padding=1)
        elif case in ("conv_wide_rowadd_silu", "conv_ragged_rowadd_silu"):
            ra = rnd(NB, N, seed=5)
            out = nv.conv3x3(x, wp, b, rowadd=ra, act=nv.ACT_SILU)
            ref = F.silu(F.conv2d(xr, w4.float(), b.float(), padding=1) + ra.float()[:, :, None, None])
        elif case == "conv_skip_segments":
            s1, s2 = rnd(NB, H, W, 96, seed=7), rnd(NB, H, W, 32, seed=8)
            ws = rnd(N, 128, scale=128 ** -0.5, seed=9)
            out = nv.conv3x3(x, torch.cat([wp, ws], 1).contiguous(), b, skip=[s1, s2])
            ref = F.conv2d(xr, w4.float(), b.float(), padding=1) + \
                F.conv2d(torch.cat([s1, s2], 3).float().permute(0, 3, 1, 2), ws.float()[:, :, None, None])
        else:
            r = rnd(NB, H, W, N, seed=3)
            out = nv.conv3x3(x, wp, b, residual=r)
            ref = F.conv2d(xr, w4.float(), b.float(), padding=1) + r.float().permute(0, 3, 1, 2)
        return out, ref.permute(0, 2, 3, 1)
    out, ref = run()
    torch.cuda.synchronize()
    close(out, ref)


@pytest.mark.parametrize("C", [64, 320])
def test_geglu(nv, C):
    M, inner = 512, 4 * C
    x = rnd(M, C)
    w = rnd(2 * inner, C, scale=C ** -0.5, seed=1)
    b = rnd(2 * inner, seed=2)
    wp, bp, bn = nv.pack_geglu(w, b)
    out = nv.linear(x, wp, bp, act=nv.ACT_GEGLU, bn_force=bn)
    torch.cuda.synchronize()
    y = (x.float() @ w.float().t() + b.float()).half()
    v, g = y.chunk(2, dim=-1)
    close(out, v.float() * F.gelu(g.float()), rtol=8e-3, atol=8e-3)


@pytest.mark.parametrize("NB,H,W,C,N", [(2, 64, 64, 320, 320), (3, 8, 8, 128, 64), (2, 32, 32, 640, 320),
                                        (8, 8, 8, 1280, 1280), (2, 8, 8, 2560, 1280),   # split-K path
                                        (1, 16, 16, 1280, 640), (2, 24, 24, 64, 128), (1, 12, 12, 64, 64),
                                        (1, 128, 128, 128, 128)])
def test_conv3x3(nv, NB, H, W, C, N):
    x = rnd(NB, H, W, C)
    w = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
    b = rnd(N, seed=2)
    emb = rnd(NB, N, seed=3)
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = nv.conv3x3(x, wp, b, rowadd=emb)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1) + emb.float()[:, :, None, None]
    close(out, ref.permute(0, 2, 3, 1))


def test_conv3x3_fused_skip(nv):
    NB, H, W, C, Cx1, Cx2, N = 2, 32, 32, 320, 640, 320, 320
    h, x1, x2 = rnd(NB, H, W, C), rnd(NB, H, W, Cx1, seed=4), rnd(NB, H, W, Cx2, seed=5)
    w = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
    ws = rnd(N, Cx1 + Cx2, scale=(Cx1 + Cx2) ** -0.5, seed=6)
    b = rnd(N, seed=2)
    wp = torch.cat([w.permute(0, 2, 3, 1).reshape(N, 9 * C), ws], dim=1).contiguous()
    out = nv.conv3x3(h, wp, b, skip=[x1, x2])
    torch.cuda.synchronize()
    ref = F.conv2d(h.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1)
    ref = ref + F.conv2d(torch.cat([x1, x2], 3).float().permute(0, 3, 1, 2), ws.float()[:, :, None, None])
    close(out, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("NB,H,W,C,N", [(2, 64, 64, 320, 320), (1, 32, 32, 64, 64), (2, 16, 16, 128, 128)])
def test_conv3x3_stride2(nv, NB, H, W, C, N):
    x = rnd(NB, H, W, C)
    w = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
    b = rnd(N, seed=2)
    wp = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = nv.conv3x3(x, wp, b, stride=2)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), padding=1, stride=2)
    close(out, ref.permute(0, 2, 3, 1))


def test_bmm_nt_headsplit(nv):
    # QK^T per (batch, head): a [B*h, M, d], b [B*h, Nk, d] -> s [B*h, M, Nk]
    BH, M, Nk, d = 16, 256, 148 + 4, 40
    a, b = rnd(BH, M, d), rnd(BH, Nk, d, seed=1)
    s = torch.empty(BH, M, Nk, device="cuda", dtype=torch.float16)
    nv.bmm_nt(a, b, out=s, so=(M * Nk, 0, 0, Nk, 0, 1))
    torch.cuda.synchronize()
    close(s, torch.bmm(a.float(), b.float().transpose(1, 2)))


def test_softmax_plain_and_bias(nv):
    B, R, Cc = 12, 144, 144
    s = rnd(B, R, Cc, scale=3.0)
    ref = torch.softmax((s.float() * 0.125).half().float(), -1)
    out = nv.softmax_(s.clone(), 0.125)
    nheads, nwin = 3, 4
    bias, mask = rnd(nheads, R, Cc, seed=2), rnd(nwin, R, Cc, seed=3)
    out2 = nv.softmax_(s.clone(), 0.125, bias=bias, nheads=nheads, mask=mask, nwin=nwin)
    torch.cuda.synchronize()
    close(out, ref, rtol=4e-3, atol=1e-4)
    b_idx = torch.arange(B, device="cuda")
    t = (s.float() * 0.125).half()
    t = (t + bias[b_idx % nheads]).half()
    t = (t + mask[(b_idx // nheads) % nwin]).half()
    close(out2, torch.softmax(t.float(), -1), rtol=4e-3, atol=1e-4)


def test_softmax_long_rows(nv):
    s = rnd(2, 64, 4096, scale=4.0)
    out = nv.softmax_(s.clone(), 512 ** -0.5)
    torch.cuda.synchronize()
    close(out, torch.softmax((s.float() * 512 ** -0.5).half().float(), -1), rtol=4e-3, atol=1e-5)


def test_timestep_embedding(nv):
    t = torch.tensor([1, 21, 501, 981], device="cuda", dtype=torch.int64)
    out = nv.timestep_embedding(t, 320)
    torch.cuda.synchronize()
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device="cuda") / half)
    args = t[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    close(out, ref, rtol=2e-3, atol=2e-3)


def test_layout_and_resample(nv):
    x = rnd(2, 8, 6, 10)  # NCHW
    nhwc = nv.nchw_to_nhwc(x, cpad=16)
    back = nv.nhwc_to_nchw(nhwc, 8, mul=0.5, add=0.5, lo=0.0, hi=1.0)
    x32 = x.float()
    nhwc32 = nv.nchw_to_nhwc(x32)
    y = rnd(2, 5, 7, 64)
    up = nv.upsample2x(y)
    col = nv.im2col3x3(rnd(2, 6, 6, 4, seed=8), 40)
    torch.cuda.synchronize()
    assert torch.equal(nhwc[..., :8], x.permute(0, 2, 3, 1)) and nhwc[..., 8:].abs().sum() == 0
    assert torch.equal(nhwc32, x.permute(0, 2, 3, 1))
    close(back, (x.float() * 0.5 + 0.5).half().float().clamp(0, 1), rtol=1e-3, atol=1e-3)
    ref_up = F.interpolate(y.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), ref_up)
    xs = rnd(2, 6, 6, 4, seed=8)
    unf = F.unfold(xs.permute(0, 3, 1, 2).float(), 3, padding=1)  # [N, C*9, L] ordered (c, tap)
    unf = unf.reshape(2, 4, 9, 36).permute(0, 3, 2, 1).reshape(2, 6, 6, 36)
    assert torch.equal(col[..., :36].float(), unf) and col[..., 36:].abs().sum() == 0


def test_window_roundtrip_and_patch_merge(nv):
    B, H, W, C, ws, shift = 2, 16, 20, 64, 12, 6
    x = rnd(B, H, W, C)
    win = nv.window_gather(x, ws, shift)
    res = rnd(B, H, W, C, seed=3)
    back = nv.window_scatter(win, B, H, W, ws, shift, res)
    pm = nv.patch_merge_gather(rnd(1, 5, 7, 64, seed=4))
    torch.cuda.synchronize()
    # reference via torch ops (swin.py:269-287)
    Hp, Wp = 24, 24
    xp = F.pad(x.float(), (0, 0, 0, Wp - W, 0, Hp - H))
    xs = torch.roll(xp, shifts=(-shift, -shift), dims=(1, 2))
    ref = xs.view(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)
    assert torch.equal(win.float(), ref)
    close(back, x.float() + res.float(), rtol=1e-3, atol=1e-3)
    y = rnd(1, 5, 7, 64, seed=4).float()
    yp = F.pad(y, (0, 0, 0, 1, 0, 1))
    refpm = torch.cat([yp[:, 0::2, 0::2], yp[:, 1::2, 0::2], yp[:, 0::2, 1::2], yp[:, 1::2, 1::2]], -1)
    assert torch.equal(pm.float(), refpm)


def test_ddim_step_matches_fp16_eager(nv):
    B = 2
    eps = rnd(2 * B, 4, 16, 16)
    x = rnd(B, 4, 16, 16, seed=1)
    coef = torch.tensor([[0.5, 0.7, 0.0, math.sqrt(0.5)], [0.9, 0.95, 0.0, math.sqrt(0.1)]],
                        device="cuda", dtype=torch.float32)
    step = torch.tensor([1], device="cuda", dtype=torch.int32)
    xp, p0 = torch.empty_like(x), torch.empty_like(x)
    nv.ddim_step(eps, x, 2.0, coef, step, xp, p0)
    torch.cuda.synchronize()
    e_u, e_c = eps.chunk(2)
    e = e_u + 2.0 * (e_c - e_u)
    a_t = torch.full((B, 1, 1, 1), 0.9, device="cuda", dtype=torch.float16)
    a_p = torch.full((B, 1, 1, 1), 0.95, device="cuda", dtype=torch.float16)
    sg = torch.full((B, 1, 1, 1), 0.0, device="cuda", dtype=torch.float16)
    s1 = torch.full((B, 1, 1, 1), math.sqrt(0.1), device="cuda", dtype=torch.float16)
    pred = (x - s1 * e) / a_t.sqrt()
    ref = a_p.sqrt() * pred + (1. - a_p - sg ** 2).sqrt() * e
    close(p0, pred, rtol=2e-3, atol=2e-3)
    close(xp, ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("B,heads,Nq,Nk,d", [(2, 8, 4096, 4096, 40), (2, 8, 4096, 148, 40), (2, 8, 1024, 1024, 80),
                                             (1, 8, 256, 256, 160), (1, 4, 100, 77, 40), (1, 8, 64, 64, 160),
                                             (1, 2, 300, 130, 64), (1, 8, 144, 576, 96)])
def test_flash_attention(nv, B, heads, Nq, Nk, d):
    from pfd_b200 import attention as att
    C = heads * d
    x = rnd(B * Nq, C, scale=1.0)
    ctx = rnd(B * Nk, C, scale=1.0, seed=3)
    wq, wk, wv = (rnd(C, C, scale=C ** -0.5, seed=s) for s in (4, 5, 6))
    q = att.project_heads(x, wq, None, B, Nq, heads, d)
    k = att.project_heads(ctx, wk, None, B, Nk, heads, d)
    vt = att.project_heads(ctx, wv, None, B, Nk, heads, d, transposed=True)
    scale = d ** -0.5
    att.USE_FLASH = True
    o_flash = att.attend(q, k, vt, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale)
    att.USE_FLASH = False
    o_unfused = att.attend(q, k, vt, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale)
    att.USE_FLASH = True
    torch.cuda.synchronize()
    qf = q[:, :Nq].float()
    kf = k[:, :Nk].float()
    vf = vt[:, :, :Nk].float().transpose(1, 2)
    s = (torch.bmm(qf, kf.transpose(1, 2)).half().float() * scale).half().float()
    ref = torch.bmm(torch.softmax(s, -1), vf).reshape(B, heads, Nq, d).permute(0, 2, 1, 3).reshape(B, Nq, C)
    close(o_unfused, ref, rtol=6e-3, atol=2e-3)
    # flash path: probabilities rounded to fp16 -> ~2^-11 relative error
    close(o_flash, ref, rtol=8e-3, atol=4e-3)
    # and against exact float64 attention with the bound derived from the kernel's arithmetic
    flash_check(o_flash.reshape(B, Nq, heads, d).permute(0, 2, 1, 3).reshape(B * heads, Nq, d), q[:, :Nq], k[:, :Nk],
                vt[:, :, :Nk].transpose(1, 2), scale, f"model B={B} h={heads} {Nq}x{Nk} d={d}")


@pytest.mark.parametrize("B,heads,Nq,Nk,d", [(8, 8, 4096, 148, 40), (2, 8, 1000, 148, 40), (3, 4, 64, 148, 40),
                                             (1, 2, 300, 77, 40), (2, 3, 130, 160, 48), (1, 5, 257, 20, 8),
                                             (1, 1, 128, 33, 16), (2, 8, 9216, 148, 40)])
def test_short_key_attention(nv, B, heads, Nq, Nk, d):
    """Cross-attention against a short context (Nk <= 160, d <= 48) through the flash kernel against an fp32 torch
    reference.  Shapes cover the BASELINE level-0 launches (512x512: 4096 queries, 768x768: 9216), ragged query
    counts, one query tile per head, partial / full last key block and the smallest head dims; one launch per call,
    a finite output everywhere (the output starts as NaN) and a relative rms error of at most 1.5e-3."""
    g = torch.Generator().manual_seed(Nq + Nk)
    q = torch.randn((B * heads, Nq, d), generator=g).cuda().half()
    Nkp = (Nk + 7) // 8 * 8
    k = torch.zeros((B * heads, Nkp, d), device="cuda", dtype=torch.float16)
    k[:, :Nk] = torch.randn((B * heads, Nk, d), generator=g).cuda().half()
    vt = torch.zeros((B * heads, d, Nkp), device="cuda", dtype=torch.float16)
    vt[:, :, :Nk] = torch.randn((B * heads, d, Nk), generator=g).cuda().half()
    scale = d ** -0.5
    out_s = torch.full((B, Nq, heads * d), float("nan"), device="cuda", dtype=torch.float16)
    nv.set_env_option(None, None)
    n0 = nv.launch_count()
    nv.flash_attn(q, k, vt, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale, out=out_s)
    assert nv.launch_count() == n0 + 1
    torch.cuda.synchronize()
    s = (torch.bmm(q.float(), k[:, :Nk].float().transpose(1, 2)).half().float() * scale).half().float()
    ref = torch.bmm(torch.softmax(s, -1), vt[:, :, :Nk].float().transpose(1, 2))
    ref = ref.reshape(B, heads, Nq, d).permute(0, 2, 1, 3).reshape(B, Nq, heads * d)
    assert torch.isfinite(out_s.float()).all()
    close(out_s, ref, rtol=8e-3, atol=4e-3)
    es = ((out_s.float() - ref).pow(2).mean() / ref.pow(2).mean()).sqrt().item()
    print(f"[short-key attention] B={B} h={heads} {Nq}x{Nk} d={d}: rel rms {es:.2e}")
    assert es < 1.5e-3


@pytest.mark.parametrize("B,heads,N,d", [(2, 8, 4096, 40), (2, 8, 1024, 80), (1, 8, 256, 160), (3, 4, 64, 40)])
def test_flash_attention_fused_qk_swapped_vt(nv, B, heads, N, d):
    """UNet self-attention path: fused q|k projection GEMM + V^T from the swapped GEMM (Wv . X^T) feeding
    the v1 flash kernel through strided views."""
    from pfd_b200 import attention as att
    C = heads * d
    x = rnd(B * N, C, scale=1.0)
    wq, wk, wv = (rnd(C, C, scale=C ** -0.5, seed=s) for s in (4, 5, 6))
    scale = d ** -0.5
    qk = att.project_heads_fused(x, torch.cat([wq, wk], 0).contiguous(), None, B, N, heads, d, 2)
    vt4 = att.project_vt_swapped(x, wv, B, N, heads, d)
    o = torch.empty((B, N, C), device="cuda", dtype=torch.float16)
    nv.flash_attn_strided(qk[:, :heads], qk[:, heads:], vt4, Nq=N, Nk=N, scale=scale, out=o)
    torch.cuda.synchronize()
    qf = (x.float() @ wq.float().t()).half().float().reshape(B, N, heads, d).permute(0, 2, 1, 3)
    kf = (x.float() @ wk.float().t()).half().float().reshape(B, N, heads, d).permute(0, 2, 1, 3)
    vf = (x.float() @ wv.float().t()).half().float().reshape(B, N, heads, d).permute(0, 2, 1, 3)
    sc = (torch.matmul(qf, kf.transpose(-1, -2)).half().float() * scale).half().float()
    ref = torch.matmul(torch.softmax(sc, -1), vf).permute(0, 2, 1, 3).reshape(B, N, C)
    close(o, ref, rtol=8e-3, atol=4e-3)
    flash_check(o.reshape(B, N, heads, d).permute(0, 2, 1, 3).reshape(B * heads, N, d),
                qk[:, :heads, :N].reshape(B * heads, N, d), qk[:, heads:, :N].reshape(B * heads, N, d),
                vt4.transpose(2, 3).reshape(B * heads, N, d), scale, f"fused q|k B={B} h={heads} N={N} d={d}")


@pytest.mark.parametrize("B,heads,Nq,Nk,d,qscale", [(2, 8, 4096, 4096, 40, 1.0), (2, 8, 1024, 148, 40, 1.0),
                                                   (1, 4, 300, 200, 64, 4.0), (1, 2, 128, 77, 8, 1.0)])
def test_flash_attention_peaked_rows(nv, B, heads, Nq, Nk, d, qscale):
    """The flash kernel on random q / k / v against an fp32 torch reference; qscale = 4 makes peaked rows (logit range
    ~ +-30: exercises the flush of small exponentials and the lazy-rescale headroom), with d = 64 and a ragged last key
    block."""
    g = torch.Generator().manual_seed(100 + Nq)
    q = (qscale * torch.randn((B * heads, Nq, d), generator=g)).cuda().half()
    Nkp = (Nk + 7) // 8 * 8
    k = torch.zeros((B * heads, Nkp, d), device="cuda", dtype=torch.float16)
    k[:, :Nk] = torch.randn((B * heads, Nk, d), generator=g).cuda().half()
    vt = torch.zeros((B * heads, d, Nkp), device="cuda", dtype=torch.float16)
    vt[:, :, :Nk] = torch.randn((B * heads, d, Nk), generator=g).cuda().half()
    scale = d ** -0.5
    out0 = torch.empty((B, Nq, heads * d), device="cuda", dtype=torch.float16)
    nv.flash_attn(q, k, vt, B=B, heads=heads, Nq=Nq, Nk=Nk, scale=scale, out=out0)
    torch.cuda.synchronize()
    s = torch.bmm(q.float(), k[:, :Nk].float().transpose(1, 2))
    if qscale == 1.0:
        s = (s.half().float() * scale).half().float()      # the reference's fp16 score tensor (attention.py:188)
    else:
        # peaked rows (|logit| ~ 30): an fp16 score tensor carries 1.6e-2 absolute logit error, i.e. percent-level
        # noise in P that is the REFERENCE's rounding, not the kernel's (fp32 logits) -> compare with exact logits
        s = s * scale
    ref = torch.bmm(torch.softmax(s, -1), vt[:, :, :Nk].float().transpose(1, 2))
    ref = ref.reshape(B, heads, Nq, d).permute(0, 2, 1, 3).reshape(B, Nq, heads * d)
    close(out0, ref, rtol=8e-3, atol=4e-3)
