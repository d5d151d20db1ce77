"""GroupNorm and LayerNorm kernels against float64 (norm_ref.py) at every thread layout of pfd_groupnorm_f16 and every
register-row size of the LayerNorm kernel, on plain data and on activations with large common offsets, constant groups
and rows, outlier pivot pixels and affine parameters with zeros, negative values and large shifts.

Every GroupNorm case runs through three statistics paths: the fast atomic kernel from a pre-zeroed scratch ring slot,
the fast kernel from a garbage-filled slot the call zeroes itself (zero_ws = 1, the ring's fallback slot), and
deterministic mode from a garbage-filled slot (it overwrites the slot).  Each output must be finite, within the
per-element bound and pass the rms check.  On a constant group the bound has no statistics term: the output must be
beta (or SiLU(beta)) to within half an fp16 ulp and the fp32 rounding of b = beta - mean * a; a constant LayerNorm row
must be beta to within one fp16 ulp.
"""
import pytest
import torch

from attention_ref import ulp16
from norm_ref import (GN_KINDS, GROUPS, LN_KINDS, gn_inputs, groupnorm_ref, layernorm_ref, ln_inputs, norm_check)

pytestmark = pytest.mark.gpu

GN_SHAPES = [  # (C1, C2, HW, NB, eps)
    (32, 0, 4096, 2, 1e-5),          # 1 channel per group: eight groups inside one 8-channel vector
    (96, 0, 1369, 2, 1e-5),          # 3 channels per group straddle the vectors; HW = 1369 leaves a ragged chunk
    (192, 0, 9, 2, 1e-6),            # 6 channels per group; 9 pixels
    (320, 0, 4096, 2, 1e-5),         # 240 threads: the deterministic fold's last warp is partial
    (512, 0, 1369, 2, 1e-6),
    (640, 0, 1024, 2, 1e-5),
    (1280, 0, 256, 2, 1e-5),
    (1280, 640, 256, 2, 1e-5),       # C = 1920 from two sources
    (2560, 0, 64, 2, 1e-5),          # 320 vectors: one pixel lane of 320 threads
    (2304, 0, 81, 2, 1e-5),          # 288 vectors
    (2688, 0, 64, 2, 1e-5),          # rows wider than the CTA: a thread walks several vectors
    (2560, 2560, 64, 1, 1e-5),       # wide rows from two sources
    (320, 640, 1024, 2, 1e-5),       # 30 channels per group: group 10 straddles the x1 / x2 boundary
    (320, 0, 1, 8, 1e-5),            # one pixel, fewer than the pixel lanes
    (128, 0, 65536, 2, 1e-6),        # 128 deterministic chunks per image
    (128, 0, 262144, 1, 1e-6),       # the VAE decoder at a 512^2 output
    (320, 0, 1024, 8, 1e-5),         # NB = 8
    (320, 0, 16, 64, 1e-5),          # NB = 64: the ring slot's and the deterministic scratch's limit
]
LN_CHANNELS = [8, 192, 256, 264, 512, 520, 1024, 1032, 2048, 2056, 4096]   # every register-row size, both sides of each
LN_ROWS = (1, 7, 9, 1000)                                                   # not multiples of the 8 rows per CTA


@pytest.fixture(scope="module")
def nv():
    from pfd_b200 import native
    native.load()
    return native


def gn_abi(nv, x1, x2, gamma, beta, eps, silu, ws, zero_ws):
    NB, HW, C1 = x1.shape
    C2 = x2.shape[-1] if x2 is not None else 0
    out = torch.empty((NB, HW, C1 + C2), device="cuda", dtype=torch.float16)
    nv._check(nv.load().pfd_groupnorm_f16(x1.data_ptr(), C1, nv._p(x2), C2, NB, HW, GROUPS, gamma.data_ptr(),
                                          beta.data_ptr(), eps, int(silu), out.data_ptr(), ws.data_ptr(), zero_ws,
                                          nv.stream_ptr()), "pfd_groupnorm_f16")
    return out


def gn_paths(nv, x1, x2, gamma, beta, eps, silu):
    """[(label, out)] of the three statistics paths."""
    import pfd_b200
    NB, HW, C1 = x1.shape
    garbage = lambda: torch.full((NB * GROUPS * 2 + NB,), float("nan"), device="cuda", dtype=torch.float64)
    nv.gn_reset()
    ring = nv.groupnorm(x1.view(NB, HW, 1, C1), gamma, beta, eps, silu=silu,
                        x2=None if x2 is None else x2.view(NB, HW, 1, -1)).view(NB, HW, -1)
    fallback = gn_abi(nv, x1, x2, gamma, beta, eps, silu, garbage(), 1)
    was = pfd_b200.is_deterministic()
    pfd_b200.set_deterministic(True)
    try:
        det = gn_abi(nv, x1, x2, gamma, beta, eps, silu, garbage(), 0)
    finally:
        pfd_b200.set_deterministic(was)
    torch.cuda.synchronize()
    return [("ring slot", ring), ("self-zeroing slot", fallback), ("deterministic", det)]


@pytest.mark.parametrize("silu", [False, True], ids=["plain", "silu"])
@pytest.mark.parametrize("kind", GN_KINDS)
@pytest.mark.parametrize("C1,C2,HW,NB,eps", GN_SHAPES)
def test_groupnorm_f64(nv, C1, C2, HW, NB, eps, kind, silu):
    x1, x2, gamma, beta, _ = gn_inputs(NB, HW, C1, C2, kind)
    x1, gamma, beta = x1.cuda(), gamma.cuda(), beta.cuda()
    x2 = x2.cuda() if x2 is not None else None
    ref, bound, var = groupnorm_ref(x1, x2, gamma, beta, eps, silu)
    label = f"GroupNorm C={C1}+{C2} HW={HW} NB={NB} eps={eps:g} {kind} silu={silu}"
    for path, out in gn_paths(nv, x1, x2, gamma, beta, eps, silu):
        norm_check(out, ref, bound, var, f"{label} [{path}]")


def ln_eps(kind):
    return 1e-6 if kind in ("const", "affine") else 1e-5


@pytest.mark.parametrize("residual", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("kind", LN_KINDS)
@pytest.mark.parametrize("C", LN_CHANNELS)
def test_layernorm_f64(nv, C, kind, residual):
    x, res, gamma, beta, const = ln_inputs(max(LN_ROWS), C, kind)
    x, res, gamma, beta = x.cuda(), res.cuda(), gamma.cuda(), beta.cuda()
    eps = ln_eps(kind)
    for rows in LN_ROWS:
        r = res[:rows] if residual else None
        out = nv.layernorm(x[:rows], gamma, beta, eps, residual=r)
        torch.cuda.synchronize()
        ref, bound, var = layernorm_ref(x[:rows], r, gamma, beta, eps)
        label = f"LayerNorm C={C} rows={rows} {kind} residual={residual}"
        norm_check(out, ref, bound, var, label)
        if kind == "const":
            cm = const[:rows].cuda().bool()
            err = (out.double() - ref)[cm].abs()
            assert bool((err <= ulp16(ref[cm])).all()), f"{label}: a constant row is off beta by {float(err.max()):.3g}"


@pytest.mark.parametrize("kind", ["random", "dc16"])
@pytest.mark.parametrize("C", LN_CHANNELS)
def test_layernorm_out_aliases_residual(nv, C, kind):
    """out == residual, as the SeeCoder query decoder calls it (lquery <- LN(attn + lquery))."""
    x, res, gamma, beta, _ = ln_inputs(max(LN_ROWS), C, kind)
    x, res, gamma, beta = x.cuda(), res.cuda(), gamma.cuda(), beta.cuda()
    ref, bound, var = layernorm_ref(x, res, gamma, beta, 1e-5)
    out = nv.layernorm(x, gamma, beta, 1e-5, residual=res, out=res)
    torch.cuda.synchronize()
    assert out.data_ptr() == res.data_ptr()
    norm_check(out, ref, bound, var, f"LayerNorm C={C} {kind} out aliasing the residual")
