"""The GEMM's staged epilogue: consumers write the fp16 tile to shared memory, the store warps add the residual and
write 16-byte chunks.  Every N tile width is forced in turn and checked against torch fp32; a second launch must
reproduce the bits."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BNS = (64, 128, 160, 192, 256)


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to("cuda", torch.float16)


def close(out, ref, rtol=4e-3, atol=4e-3):
    err = (out.float() - ref.float()).abs()
    bad = (err > atol + rtol * ref.float().abs()).sum().item()
    assert bad == 0, f"{bad}/{err.numel()} mismatches, max err {err.max().item():.4g}"


def conv(nv, x, wp, N, bn, **kw):
    NB, H, W, C = x.shape
    out = torch.empty((NB, H, W, N), device="cuda", dtype=torch.float16)
    nv.gemm_raw([(x, 9, C, (x.stride(2), x.stride(1), x.stride(0)))], in_w=W, in_h=H, stride=1, W=W, H=H, NB=NB,
                w=wp, N=N, K=wp.stride(0), out=out, so=(out.stride(0), 0, out.stride(1), out.stride(2), 0, 1),
                bn_force=bn, **kw)
    return out


def case_data(nv, case, bn):
    """(run, ref): run() launches the GEMM and returns its output, ref is the fp32 result."""
    if case == "linear_ragged_bias_res":               # M not a multiple of 128, N not a multiple of any tile
        x, w, b, r = rnd(1000, 192), rnd(328, 192, scale=192 ** -0.5, seed=1), rnd(328, seed=2), rnd(1000, 328, seed=3)
        return (lambda: nv.linear(x, w, b, residual=r, bn_force=bn),
                x.float() @ w.float().t() + b.float() + r.float())
    if case == "linear_inplace_res":                   # out is the residual tensor (x = x + f(x) in place)
        x, w, b, r = rnd(700, 320), rnd(320, 320, scale=320 ** -0.5, seed=1), rnd(320, seed=2), rnd(700, 320, seed=3)

        def run():
            o = r.clone()
            return nv.linear(x, w, b, residual=o, out=o, bn_force=bn)
        return run, x.float() @ w.float().t() + b.float() + r.float()
    if case == "persistent_many_tiles":               # several tiles per CTA: the staging buffer is reused
        M = 16384 + 72
        x, w, b, r = rnd(M, 64), rnd(320, 64, scale=0.125, seed=1), rnd(320, seed=2), rnd(M, 320, seed=3)
        return (lambda: nv.linear(x, w, b, residual=r, bn_force=bn),
                x.float() @ w.float().t() + b.float() + r.float())
    if case == "geglu":
        M, C, inner = 300, 320, 1920                    # 2 * inner is a multiple of every tile width
        x, w, b = rnd(M, C), rnd(2 * inner, C, scale=C ** -0.5, seed=1), rnd(2 * inner, seed=2)
        h = bn // 2
        tile = torch.arange(2 * inner // bn, device="cuda").reshape(-1, 1)
        j = torch.arange(h, device="cuda").reshape(1, -1)
        src = torch.stack([tile * h + j, inner + tile * h + j], dim=1).reshape(-1)
        wp, bp = w.index_select(0, src).contiguous(), b.index_select(0, src).contiguous()
        y = (x.float() @ w.float().t() + b.float()).half()
        v, g = y.chunk(2, dim=-1)
        return lambda: nv.linear(x, wp, bp, act=nv.ACT_GEGLU, bn_force=bn), v.float() * F.gelu(g.float())
    if case == "head_split_bias_res":                 # [B, tokens, heads*d] -> [B, heads, tokens, d] (cdiv = d)
        B, T, heads, d = 2, 200, 5, 64
        x, w, b = rnd(B * T, 256), rnd(heads * d, 256, scale=1 / 16, seed=1), rnd(heads * d, seed=2)
        r = rnd(B, heads, T, d, seed=3)

        def run():
            out = torch.empty((B, heads, T, d), device="cuda", dtype=torch.float16)
            nv.gemm_raw([(x, 1, 256, (256, 256 * T, 256 * T))], in_w=T, in_h=1, stride=1, W=T, H=1, NB=B, w=w,
                        N=heads * d, K=256, bias=b, residual=r, out=out, so=(heads * T * d, 0, 0, d, T * d, 1),
                        ndiv=1, cdiv=d, bn_force=bn)
            return out
        y = (x.float() @ w.float().t() + b.float()).reshape(B, T, heads, d).permute(0, 2, 1, 3)
        return run, y + r.float()
    NB, H, W, C, N = 3, 24, 20, 64, 200                 # conv raster with padded pixel tiles
    x = rnd(NB, H, W, C)
    w4 = rnd(N, C, 3, 3, scale=(9 * C) ** -0.5, seed=1)
    b = rnd(N, seed=2)
    wp = w4.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w4.float(), b.float(), padding=1)
    if case == "conv_rowadd_silu":
        ra = rnd(NB, N, seed=5)
        return (lambda: conv(nv, x, wp, N, bn, bias=b, rowadd=ra, act=nv.ACT_SILU),
                F.silu(ref + ra.float()[:, :, None, None]).permute(0, 2, 3, 1))
    r = rnd(NB, H, W, N, seed=3)
    return lambda: conv(nv, x, wp, N, bn, bias=b, residual=r), ref.permute(0, 2, 3, 1) + r.float()


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("case", ["linear_ragged_bias_res", "linear_inplace_res", "persistent_many_tiles", "geglu",
                                  "head_split_bias_res", "conv_rowadd_silu", "conv_bias_res"])
def test_staged_epilogue(nv, case, bn):
    run, ref = case_data(nv, case, bn)
    a = run().clone()
    b = run().clone()
    torch.cuda.synchronize()
    close(a, ref, *((8e-3, 8e-3) if case == "geglu" else ()))
    assert torch.equal(a, b), "two launches gave different bits"
