"""Float64 references, error bounds, seeded inputs and kernel emulators for the annotator layer-kernel tests
(test_annotator_kernels_gpu.py and its CPU model test_annotator_kernels_model_cpu.py).  This module holds no tests.

Every layer kernel of the PiDiNet, M-LSD and OpenPose networks, plus the shared ToPILImage quantiser (``to_u8`` in
pfd_b200/csrc/common.h), is restated here from its contract, in float64 torch on whatever device the inputs live on:

* ``*_ref`` return the exact result (float64) and, where the kernel rounds, a per-element bound derived from its
  arithmetic: one fp16 rounding of the result where the output is fp16 (``f16_bound``), ``n * u * sum|w x|`` for an
  fp32 sum of n terms (u = 2^-24; 2^-23 per term for the tensor-core accumulation, which may truncate), and the
  documented 2-ulp error of expf where the kernel uses it.
* Integer cases use small-integer or dyadic inputs and weights, so that every product and partial sum is exact in fp32
  and the result exact in the output type: the kernel must then equal the reference bit for bit, in any summation
  order.
* ``*_model`` are numpy float32 (or float64-summed) emulations of the kernels' arithmetic and index rules, with a
  ``mutant`` switch for the subtly wrong variants listed in ``MUTANTS``.  The CPU model test shows that the emulations
  pass every check and that each mutant fails at least one.
"""
import numpy as np
import torch
import torch.nn.functional as F

from attention_ref import ulp16

U32 = 2.0 ** -24             # fp32 unit roundoff
F32 = np.float32
D = 24                       # CDCM / CSAM / MapReduce width
DILATIONS = (5, 7, 9, 11)
SIDE_PARAMS = 4 * D + 4 + 36 + D + 1
FUSE_TOL = 1e-9              # |pre - integer| below which a fuse level may truncate either way (the kernel's float64
                             # classifier and exp differ from numpy's by ~1e-13 of the 0..255 range)
HED_NORM = (104.00698793, 116.66876762, 122.67891434)    # a non-integer per-channel mean, as HED's learned `norm`
HED_SCALE = 1.0 / 255.0

MUTANTS = {
    "dw_drop_last_col": "depthwise conv without its last-column tap",
    "ceil_pool": "2x2 max-pool with ceil instead of floor",
    "mlsd_sym_pad": "M-LSD stride 2 with symmetric padding 1 instead of TFLite's (0, 1, 0, 1)",
    "mlsd_relu6_out_only": "M-LSD depthwise ReLU6 on the output only, no min(x, 6) on the input",
    "upsample_align_false": "upsample with align_corners=False",
    "csam_pad_u": "CSAM zero-padding u instead of y",
    "cdcm_swap_dilations": "CDCM with dilations 5 and 7 swapped",
    "cdcm_pack_lanes_swapped": "pack_cdcm with lanes g and t exchanged",
    "quant_fp32_product": "quantiser product rounded in fp32",
    "fuse_unclamped_i1": "fuse with an unclamped second bilinear index",
    "head_relu_paf": "ReLU applied to the PAF head",
}


# ------------------------------------------------------------------------------------------------- helpers
def gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def ints(shape, lo: int, hi: int, seed: int, scale: float = 1.0) -> torch.Tensor:
    """float64 integers in [lo, hi] times scale (a power of two: the values stay exact in fp16)."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=gen(seed)).double() * scale


def randn(shape, seed: int, scale: float = 1.0) -> torch.Tensor:
    shape = (shape,) if isinstance(shape, int) else tuple(shape)
    return torch.randn(shape, generator=gen(seed), dtype=torch.float64) * scale


def rand(shape, seed: int, lo: float, hi: float) -> torch.Tensor:
    return lo + (hi - lo) * torch.rand(tuple(shape), generator=gen(seed), dtype=torch.float64)


def f16_bound(ref: torch.Tensor, d: torch.Tensor) -> torch.Tensor:
    """Bound of |fp16(v) - ref| when |v - ref| <= d: d plus half an fp16 ulp at |ref| + d."""
    return 0.5 * ulp16(ref.abs() + d) + d


def err_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound (0 where both are 0, inf where the bound is 0 and the error is not)."""
    e = (out.double() - ref.double()).abs()
    r = torch.where(e == 0, torch.zeros_like(e), e / bound.double())
    return float(r.max()) if r.numel() else 0.0


def mismatches(out: torch.Tensor, ref: torch.Tensor) -> int:
    """Elements that differ in value (a shape mismatch counts as all of them)."""
    if tuple(out.shape) != tuple(ref.shape):
        return max(out.numel(), ref.numel(), 1)
    return int((out.double() != ref.double()).sum())


def bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    w = {2: torch.int16, 4: torch.int32, 1: torch.uint8}[a.element_size()]
    return torch.equal(a.contiguous().view(w), b.contiguous().view(w))


def nchw(x):
    return x.permute(0, 3, 1, 2)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def fma32(a, b, c):
    """float32 fused multiply-add: the float64 product of two float32 values is exact."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def np32(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().float().numpy()


# ------------------------------------------------------------------------------------------------- quantiser
def quant_inputs_f16() -> torch.Tensor:
    """The 15 361 fp16 values in [0, 1] (bit patterns 0 .. 0x3C00)."""
    return torch.arange(0x3C01, dtype=torch.int16).view(torch.float16)


def quant_inputs_f32() -> torch.Tensor:
    """float32 k/255 (k = 0..255), one ulp either side of each, and 1.0; all in [0, 1]."""
    v = (np.arange(256, dtype=np.float64) / 255.0).astype(F32)
    x = np.concatenate([v, np.nextafter(v, F32(-1)), np.nextafter(v, F32(2)), [F32(1)]])
    return torch.from_numpy(np.unique(x[(x >= 0) & (x <= 1)]))


def to_u8_ref(x: torch.Tensor) -> torch.Tensor:
    """ToPILImage's pic.mul(255).byte() in the input's dtype, on the CPU (uint8)."""
    return x.cpu().mul(255).byte()


def to_u8_model(x: torch.Tensor, mutant=None) -> torch.Tensor:
    """The kernel's to_u8: the product rounded in the input's dtype (fp16: __hmul), truncated, low 8 bits."""
    v = np32(x)
    p = (v * F32(255)).astype(F32)
    if x.dtype == torch.float16 and mutant != "quant_fp32_product":
        p = p.astype(np.float16).astype(F32)
    return torch.from_numpy(p.astype(np.int64).astype(np.uint8))


def as_image(vals: torch.Tensor, B: int = 1):
    """A flat value list -> NCHW [B, 3, 1, W] image (padded with zeros), and the number of real values."""
    n = vals.numel()
    W = -(-n // (3 * B))
    img = torch.zeros(B * 3 * W, dtype=vals.dtype)
    img[:n] = vals
    return img.reshape(B, 3, 1, W), n


def hed_input_ref(x: torch.Tensor, norm, scale: float, cpad: int) -> torch.Tensor:
    """[B,3,H,W] image -> fp16 [B,H,W,cpad]: fp16((u8 - norm) * scale) with both operations in fp32, pad channels 0."""
    u = to_u8_ref(x).float()
    nm = torch.tensor(norm, dtype=torch.float32).view(1, 3, 1, 1)
    v = ((u - nm) * torch.tensor(scale, dtype=torch.float32)).half()
    B, _, H, W = x.shape
    out = torch.zeros((B, H, W, cpad), dtype=torch.float16)
    out[..., :3] = nhwc(v)
    return out


def mlsd_input_ref(x: torch.Tensor) -> torch.Tensor:
    """[B,3,H,W] image -> fp16 [B,H,W,16] = [u8 - 127.5 (rgb), 1 - 127.5, 0 x 12]."""
    u = to_u8_ref(x).float() - 127.5
    B, _, H, W = x.shape
    out = torch.zeros((B, H, W, 16), dtype=torch.float16)
    out[..., :3] = nhwc(u).half()
    out[..., 3] = -126.5
    return out


# ------------------------------------------------------------------------------------------------- pools, im2col
def pool_ref(x: torch.Tensor) -> torch.Tensor:
    """F.max_pool2d(2) (floor) of channel-last fp16 x, exact."""
    return nhwc(F.max_pool2d(nchw(x.float()), 2)).half()


def pool_model(x: torch.Tensor, mutant=None) -> torch.Tensor:
    """The kernels' 2x2 max of channel-last fp16 x; mutant 'ceil_pool' keeps the odd last row / column."""
    v = np32(x)
    B, H, W, C = v.shape
    if mutant == "ceil_pool":
        Ho, Wo = -(-H // 2), -(-W // 2)
        p = np.full((B, 2 * Ho, 2 * Wo, C), -np.inf, F32)
        p[:, :H, :W] = v
        v = p
    else:
        Ho, Wo = H // 2, W // 2
        v = v[:, :2 * Ho, :2 * Wo]
    m = np.maximum(np.maximum(v[:, 0::2, 0::2], v[:, 0::2, 1::2]), np.maximum(v[:, 1::2, 0::2], v[:, 1::2, 1::2]))
    return torch.from_numpy(np.ascontiguousarray(m).astype(np.float16))


def im2col7_ref(x: torch.Tensor) -> torch.Tensor:
    """F.unfold(7, padding=3) of channel-last x, reordered to rows [B*H*W] of k = tap * C + c."""
    B, H, W, C = x.shape
    u = F.unfold(nchw(x.float()), 7, padding=3)                     # [B, C*49, H*W], row c*49 + tap
    u = u.reshape(B, C, 49, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 49 * C)
    return u.half()


# ------------------------------------------------------------------------------------------------- PiDiNet
def dw_weights(w4: torch.Tensor) -> torch.Tensor:
    """[C, 1, ks, ks] -> the kernels' fp32 tap-major [ks*ks, C]."""
    return w4.reshape(w4.shape[0], -1).t().float().contiguous()


def pidinet_dw_ref(x: torch.Tensor, w4: torch.Tensor, pool: bool):
    """relu(depthwise conv2d(padding ks//2)) of x (after max_pool2d(2) when pool), float64 NHWC -> (out, bound,
    pooled float64 or None)."""
    C, ks = w4.shape[0], w4.shape[-1]
    p = nchw(x.double())
    if pool:
        p = F.max_pool2d(p, 2)
    w = w4.double().to(x.device)
    out = F.relu(F.conv2d(p, w, padding=ks // 2, groups=C))
    absd = F.conv2d(p.abs(), w.abs(), padding=ks // 2, groups=C)
    bound = f16_bound(out, ks * ks * U32 * absd)
    return nhwc(out), nhwc(bound), (nhwc(p) if pool else None)


def pidinet_dw_model(x: torch.Tensor, wt: torch.Tensor, pool: bool, mutant=None):
    """pidinet_dw_kernel: fp32 fmas in (ky, kx) order over the (pooled) fp16 input, ReLU, one fp16 rounding."""
    pooled = pool_model(x, mutant) if pool else x.cpu()
    v = np32(pooled)
    w = np32(wt)
    ks = {9: 3, 25: 5}[w.shape[0]]
    R = ks // 2
    B, h, wd, C = v.shape
    vp = np.zeros((B, h + 2 * R, wd + 2 * R, C), F32)
    vp[:, R:R + h, R:R + wd] = v
    acc = np.zeros((B, h, wd, C), F32)
    for ky in range(ks):
        for kx in range(ks):
            if mutant == "dw_drop_last_col" and kx == ks - 1:
                continue
            acc = fma32(vp[:, ky:ky + h, kx:kx + wd], w[ky * ks + kx], acc)
    out = torch.from_numpy(np.maximum(acc, F32(0)).astype(np.float16))
    return (out, pooled) if pool else out


def reduce_ref(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor):
    """m = b + relu(x) @ w (x [..., C], w [C, 24]) in float64 -> (m, bound of the fp16 output)."""
    C = x.shape[-1]
    r = F.relu(x.double())
    wd, bd = w.double().to(x.device), b.double().to(x.device)
    m = r @ wd + bd
    d = (C + 1) * U32 * (r @ wd.abs() + bd.abs())
    return m, f16_bound(m, d)


def reduce_model(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    v = np.maximum(np32(x), F32(0))
    wn, bn = np32(w), np32(b)
    acc = np.broadcast_to(bn, v.shape[:-1] + (D,)).astype(F32)
    for c in range(v.shape[-1]):
        acc = fma32(v[..., c:c + 1], wn[c], acc)
    return torch.from_numpy(acc.astype(np.float16))


def cdcm_ref(m: torch.Tensor, Ws: torch.Tensor):
    """u = sum_d conv2d(m, W_d, padding=d, dilation=d), d = 5, 7, 9, 11; m [B,h,w,24], Ws [4, 24, 24, 3, 3] ->
    (u float64 NHWC, bound of the tensor-core fp32 accumulation over K = 864)."""
    mi = nchw(m.double())
    W = Ws.double().to(m.device)
    u = sum(F.conv2d(mi, W[j], padding=d, dilation=d) for j, d in enumerate(DILATIONS))
    a = sum(F.conv2d(mi.abs(), W[j].abs(), padding=d, dilation=d) for j, d in enumerate(DILATIONS))
    return nhwc(u), nhwc(864 * 2.0 ** -23 * a)


def pack_cdcm_lanes_swapped(weights) -> torch.Tensor:
    """pidinet.pack_cdcm with lane t*8 + g instead of g*4 + t (a mutant)."""
    w = torch.stack([x.detach().float() for x in weights])
    k = w.permute(0, 3, 4, 2, 1).reshape(54, 2, 4, 2, 3, 8)            # [s, hi, t, e, j, g]
    return k.permute(0, 4, 2, 5, 1, 3).reshape(54, 3, 32, 4).to(torch.float16).contiguous()


def cdcm_unpack(wpk: torch.Tensor) -> torch.Tensor:
    """Packed fragments -> dense B [864, 24] by the mma.m16n8k16 B-fragment rule the kernel relies on: lane 4g + t of
    n-tile j holds column 8j + g at step rows 2t, 2t+1 (b0) and 2t+8, 2t+9 (b1)."""
    f = wpk.cpu().double().reshape(54, 3, 8, 4, 2, 2)                   # [s, j, g, t, hi, e]
    return f.permute(0, 4, 3, 5, 1, 2).reshape(864, D)                  # K = 16s + 8hi + 2t + e, N = 8j + g


def cdcm_model(m: torch.Tensor, wpk: torch.Tensor, mutant=None) -> torch.Tensor:
    """pidinet_cdcm_kernel's implicit GEMM: K walked tap-major (dilation, ky, kx) then channel, A gathered with zero
    padding, B from the packed fragments; summed in float64, rounded to fp32."""
    dil = (7, 5, 9, 11) if mutant == "cdcm_swap_dilations" else DILATIONS
    B, h, w, _ = m.shape
    P = 11
    mp = F.pad(m.cpu().double(), (0, 0, P, P, P, P))
    cols = [mp[:, P + (ky - 1) * d:P + (ky - 1) * d + h, P + (kx - 1) * d:P + (kx - 1) * d + w]
            for d in dil for ky in range(3) for kx in range(3)]
    return (torch.cat(cols, -1) @ cdcm_unpack(wpk)).float()


def side_params(seed: int, b1_scale: float = 8.0) -> torch.Tensor:
    """CSAM conv1 w [4][24], conv1 b [4] (large, so the border padding matters), conv2 w [4][9], MapReduce w [24], b."""
    p = torch.cat([randn(4 * D, seed, 0.3), randn(4, seed + 1, b1_scale), randn(36, seed + 2, 0.3),
                   randn(D, seed + 3, 0.3), randn(1, seed + 4)])
    return p.float()


def _split_params(prm: torch.Tensor):
    p = prm.double()
    w1, b1 = p[:96].reshape(4, D), p[96:100]
    w2, wr, br = p[100:136].reshape(4, 9), p[136:160], p[160:161]
    return w1, b1, w2, wr, br


def side_ref(u: torch.Tensor, prm: torch.Tensor):
    """model.py's CSAM + MapReduce in float64: y = conv1x1(relu(u)) + b1; a = sigmoid(conv3x3(y, padding 1));
    side = conv1x1(u * a) + br -> (side [B,h,w], bound of the kernel's fp32 evaluation)."""
    w1, b1, w2, wr, br = (t.to(u.device) for t in _split_params(prm))
    ui = nchw(u.double())
    r = F.relu(ui)
    y = F.conv2d(r, w1.view(4, D, 1, 1), b1)
    W2 = w2.view(1, 4, 3, 3)
    z = F.conv2d(y, W2, padding=1)
    a = torch.sigmoid(z)
    side = F.conv2d(ui * a, wr.view(1, D, 1, 1), br)
    dy = 25 * U32 * (b1.abs().view(1, 4, 1, 1) + F.conv2d(r, w1.abs().view(4, D, 1, 1)))
    dz = 36 * U32 * F.conv2d(y.abs(), W2.abs(), padding=1) + F.conv2d(dy, W2.abs(), padding=1)
    da = 0.25 * dz + 6 * U32 * a                          # sigmoid' <= 1/4; expf (2 ulp), 1 + e and the quotient
    E = F.conv2d(ui.abs(), wr.abs().view(1, D, 1, 1))
    bound = a * 24 * U32 * E + E * da + U32 * (a * E + br.abs())
    return side[:, 0], bound[:, 0]


def side_model(u: torch.Tensor, prm: torch.Tensor, mutant=None) -> torch.Tensor:
    """pidinet_side_kernel in float32: per tap y_c = b1 + w1 . relu(u) (fmas), z += w2 * y_c inside the image only
    (mutant 'csam_pad_u': outside too, from zero u), a = 1 / (1 + exp(-z)), side = fma(a, wr . u, br)."""
    un = np32(u)
    w1, b1, w2, wr, br = (t.float().numpy() for t in _split_params(prm))
    B, h, w, _ = un.shape
    up = np.zeros((B, h + 2, w + 2, D), F32)
    up[:, 1:h + 1, 1:w + 1] = un
    inside = np.zeros((B, h + 2, w + 2), bool)
    inside[:, 1:h + 1, 1:w + 1] = True
    z = np.zeros((B, h, w), F32)
    for tap in range(9):
        ty, tx = tap // 3, tap % 3
        q = np.maximum(up[:, ty:ty + h, tx:tx + w], F32(0))
        ok = inside[:, ty:ty + h, tx:tx + w] | (mutant == "csam_pad_u")
        for c in range(4):
            yc = np.full((B, h, w), b1[c], F32)
            for k in range(D):
                yc = fma32(w1[c, k], q[..., k], yc)
            z = np.where(ok, fma32(w2[c, tap], yc, z), z)
    a = (F32(1) / (F32(1) + np.exp(-z).astype(F32))).astype(F32)
    e = np.zeros((B, h, w), F32)
    for k in range(D):
        e = fma32(wr[k], un[..., k], e)
    return torch.from_numpy(fma32(a, e, br[0]))


def fuse_sizes(H: int, W: int):
    """Side-map sizes of the network at an H x W input: stage 1 at full size, then three 2x2 floor pools."""
    return [(H >> k, W >> k) for k in range(4)]


def _coords(dst: int, src: int, clamp: bool = True):
    scale = F32(src) / F32(dst)
    d = np.arange(dst, dtype=F32) + F32(0.5)
    pos = np.maximum(fma32(d, scale, F32(-0.5)), F32(0))
    i0 = pos.astype(np.int64)
    lam = (pos - i0.astype(F32)).astype(F32)
    return i0, (np.minimum(i0 + 1, src - 1) if clamp else i0 + 1), lam


def resize_model(s: np.ndarray, H: int, W: int, mutant=None) -> np.ndarray:
    """The fuse kernel's resize_bilinear_pt on one float32 [h, w] map, reading it as flat memory with zeros past its
    end (mutant 'fuse_unclamped_i1': the second index left unclamped reads the next row / past the map)."""
    clamp = mutant != "fuse_unclamped_i1"
    h, w = s.shape
    flat = np.concatenate([s.reshape(-1), np.zeros(w + 1, F32)])
    lerp = lambda a0, a1, lam: fma32(a0, F32(1) - lam, (a1 * lam).astype(F32))      # noqa: E731
    ys, xs = np.arange(H), np.arange(W)
    if w != W:
        x0, x1, lx = _coords(W, w, clamp)
    if h != H:
        y0, y1, ly = _coords(H, h, clamp)
    else:
        y0 = y1 = ys
        ly = np.zeros(H, F32)

    def row(r):                                                       # [H] rows -> [H, W] width-pass values
        if w == W:
            return flat[r[:, None] * w + xs[None, :]]
        return lerp(flat[r[:, None] * w + x0[None, :]], flat[r[:, None] * w + x1[None, :]], lx[None, :])
    t0 = row(y0)
    if h == H:
        return t0
    return lerp(t0, row(y1), ly[:, None])


def fuse_ref(sides, cls: torch.Tensor, H: int, W: int):
    """Levels (uint8 [B,H,W]) and float64 pre-truncation values 255 * sigmoid(cb + sum c_k e_k) of the fuse, with e_k
    the side maps resized by oracle.pidinet_oracle.resize_bilinear (PyTorch's bilinear rule, align_corners=False)."""
    from oracle.pidinet_oracle import resize_bilinear
    return _fuse_levels([[resize_bilinear(np32(s[n]), H, W) for s in sides] for n in range(sides[0].shape[0])], cls)


def fuse_model(sides, cls: torch.Tensor, H: int, W: int, mutant=None):
    return _fuse_levels([[resize_model(np32(s[n]), H, W, mutant) for s in sides] for n in range(sides[0].shape[0])],
                        cls)


def _fuse_levels(es, cls):
    c = cls.double().cpu().numpy()
    pre = []
    for e in es:
        a = c[4] + c[0] * e[0].astype(np.float64) + c[1] * e[1] + c[2] * e[2] + c[3] * e[3]
        pre.append(np.clip(255.0 / (1.0 + np.exp(-a)), 0.0, 255.0))
    pre = np.stack(pre)
    return torch.from_numpy(pre.astype(np.uint8)), torch.from_numpy(pre)


def fuse_check(out: torch.Tensor, levels: torch.Tensor, pre: torch.Tensor):
    """(levels of out that differ from the reference away from an integer, pixels within FUSE_TOL of an integer,
    whether out is exactly level / 255 on all three channels)."""
    out = out.cpu()
    got = torch.round(out[:, 0].double() * 255).to(torch.int64)
    exact = all(bits_equal(out[:, k], got.float() / 255) for k in range(3))
    near = (pre - torch.round(pre)).abs() <= FUSE_TOL
    bad = int(((got != levels.long()) & ~near).sum())
    return bad, int(near.sum()), exact


# ------------------------------------------------------------------------------------------------- M-LSD
def mlsd_dw_ref(x: torch.Tensor, w4: torch.Tensor, b: torch.Tensor, stride: int):
    """clamp(conv(min(x, 6)) + b, 0, 6) float64; stride 2: F.pad(0, 1, 0, 1), padding 0; stride 1: padding 1 ->
    (out NHWC, bound of the fp16 output)."""
    C = w4.shape[0]
    xi = nchw(x.double()).clamp(max=6)
    w = w4.double().to(x.device)
    bd = b.double().to(x.device)
    if stride == 2:
        xi = F.pad(xi, (0, 1, 0, 1))
        acc, absd = F.conv2d(xi, w, stride=2, groups=C), F.conv2d(xi.abs(), w.abs(), stride=2, groups=C)
    else:
        acc, absd = F.conv2d(xi, w, padding=1, groups=C), F.conv2d(xi.abs(), w.abs(), padding=1, groups=C)
    out = (acc + bd.view(1, C, 1, 1)).clamp(0, 6)
    d = 10 * U32 * (absd + bd.abs().view(1, C, 1, 1))
    return nhwc(out), nhwc(f16_bound(out, d))


def mlsd_dw_model(x: torch.Tensor, wt: torch.Tensor, b: torch.Tensor, stride: int, mutant=None) -> torch.Tensor:
    """mlsd_dw_kernel: fmas over taps t = 0..8 of min(x, 6) at (S y + t/3 + off, S x + t%3 + off), off = -1 for
    stride 1 and 0 for stride 2 (zero outside), then clamp(acc + b, 0, 6) and one fp16 rounding."""
    v = np32(x)
    if mutant != "mlsd_relu6_out_only":
        v = np.minimum(v, F32(6))
    w, bn = np32(wt), np32(b)
    B, H, W, C = v.shape
    Ho, Wo = H // stride, W // stride
    off = -1 if (stride == 1 or mutant == "mlsd_sym_pad") else 0
    vp = np.zeros((B, H + 4, W + 4, C), F32)
    vp[:, 2:H + 2, 2:W + 2] = v
    acc = np.zeros((B, Ho, Wo, C), F32)
    for t in range(9):
        y0, x0 = t // 3 + off + 2, t % 3 + off + 2
        acc = fma32(vp[:, y0:y0 + stride * Ho:stride, x0:x0 + stride * Wo:stride], w[t], acc)
    return torch.from_numpy(np.clip((acc + bn).astype(F32), F32(0), F32(6)).astype(np.float16))


def _ac_axis(n: int, align: bool = True):
    """PyTorch's bilinear source rule for a x2 upsample in float32: align_corners=True scale (n-1)/(2n-1), src =
    scale * d; index = trunc, lambdas in float32, second index clamped.  align=False: the align_corners=False rule."""
    No = 2 * n
    d = np.arange(No, dtype=F32)
    if align:
        s = F32(n - 1) / F32(No - 1) if No > 1 else F32(0)
        f = (s * d).astype(F32)
    else:
        f = np.maximum(fma32(d + F32(0.5), F32(n) / F32(No), F32(-0.5)), F32(0))
    i0 = f.astype(np.int64)
    l1 = (f - i0.astype(F32)).astype(F32)
    return i0, np.minimum(i0 + 1, n - 1), F32(1) - l1, l1


def upsample_ref(x: torch.Tensor):
    """F.interpolate(scale_factor=2, bilinear, align_corners=True) of channel-last x in float64 from PyTorch's float32
    indices and lambdas -> (out [B,2h,2w,C], bound: 4 fp32 roundings of sum lambda |v| plus the fp16 rounding)."""
    B, h, w, C = x.shape
    iy0, iy1, ly0, ly1 = (torch.from_numpy(np.asarray(a)).to(x.device) for a in _ac_axis(h))
    ix0, ix1, lx0, lx1 = (torch.from_numpy(np.asarray(a)).to(x.device) for a in _ac_axis(w))
    v = x.double()
    ly0, ly1 = ly0.double().view(1, -1, 1, 1), ly1.double().view(1, -1, 1, 1)
    lx0, lx1 = lx0.double().view(1, 1, -1, 1), lx1.double().view(1, 1, -1, 1)

    def at(yi, xi, t):
        return t[:, yi][:, :, xi]
    out = ly0 * (lx0 * at(iy0, ix0, v) + lx1 * at(iy0, ix1, v)) + ly1 * (lx0 * at(iy1, ix0, v) + lx1 * at(iy1, ix1, v))
    a = v.abs()
    s = ly0 * (lx0 * at(iy0, ix0, a) + lx1 * at(iy0, ix1, a)) + ly1 * (lx0 * at(iy1, ix0, a) + lx1 * at(iy1, ix1, a))
    return out, f16_bound(out, 4 * U32 * s)


def upsample_model(x: torch.Tensor, mutant=None) -> torch.Tensor:
    align = mutant != "upsample_align_false"
    v = np32(x)
    B, h, w, C = v.shape
    iy0, iy1, ly0, ly1 = _ac_axis(h, align)
    ix0, ix1, lx0, lx1 = _ac_axis(w, align)
    ly0, ly1 = ly0[None, :, None, None], ly1[None, :, None, None]
    lx0, lx1 = lx0[None, None, :, None], lx1[None, None, :, None]
    at = lambda yi, xi: v[:, yi][:, :, xi]                           # noqa: E731
    top = (lx0 * at(iy0, ix0)).astype(F32) + (lx1 * at(iy0, ix1)).astype(F32)
    bot = (lx0 * at(iy1, ix0)).astype(F32) + (lx1 * at(iy1, ix1)).astype(F32)
    out = (ly0 * top.astype(F32)).astype(F32) + (ly1 * bot.astype(F32)).astype(F32)
    return torch.from_numpy(out.astype(F32).astype(np.float16))


# ------------------------------------------------------------------------------------------------- 1x1 heads
def head_ref(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, relu: bool):
    """act(b + w . x) planar float64 [B,N,h,w] (x [B,h,w,C], w [N,C]) and the fp32 bound (C + 1) u (|b| + sum|w x|)."""
    C = x.shape[-1]
    v = x.double()
    wd, bd = w.double().to(x.device), b.double().to(x.device)
    out = v @ wd.t() + bd
    if relu:
        out = F.relu(out)
    d = (C + 1) * U32 * (v.abs() @ wd.abs().t() + bd.abs())
    return nchw(out), nchw(d)


def head_model(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, relu: bool, mutant=None) -> torch.Tensor:
    """The head kernels: acc = b, fmas over the channels in order, optional ReLU; planar fp32 [B,N,h,w]."""
    v, wn, bn = np32(x), np32(w), np32(b)
    acc = np.broadcast_to(bn, v.shape[:-1] + (wn.shape[0],)).astype(F32)
    for c in range(v.shape[-1]):
        acc = fma32(v[..., c:c + 1], wn[:, c], acc)
    if relu or mutant == "head_relu_paf":
        acc = np.maximum(acc, F32(0))
    return torch.from_numpy(np.ascontiguousarray(acc.transpose(0, 3, 1, 2)))


# ------------------------------------------------------------------------------------------------- cases
# Shapes where index arithmetic goes wrong: maps smaller than the kernel window, odd sizes (floor pools, stride 2's
# extra row), the network's channel counts and 8-channel vector tails.  The GPU test runs all of them; the CPU model
# test runs the emulations through them too.
POOL_CASES = [(1, 2, 2, 8), (1, 3, 3, 8), (1, 3, 2, 8), (2, 2, 7, 16), (1, 5, 3, 128), (2, 9, 11, 64), (1, 12, 13, 136)]
IM2COL_CASES = [(1, 1, 1, 8), (1, 1, 9, 8), (2, 3, 8, 128), (1, 7, 7, 136), (1, 8, 11, 8), (2, 9, 2, 136),
                (1, 10, 10, 128)]
DW_CASES = [  # (B, H, W, C, ks, pool)
    (1, 1, 1, 8, 3, False), (1, 3, 4, 16, 5, False), (2, 4, 2, 8, 5, False), (1, 2, 1, 8, 5, False),
    (1, 13, 17, 64, 3, False), (2, 9, 11, 64, 5, False), (1, 16, 15, 240, 5, False), (2, 10, 7, 120, 3, False),
    (1, 7, 9, 64, 3, True), (2, 2, 2, 8, 3, True), (1, 3, 3, 16, 3, True), (1, 2, 5, 8, 3, True),
    (1, 5, 2, 8, 3, True), (2, 33, 31, 128, 3, True), (1, 65, 48, 240, 3, True)]
MLSD_DW_CASES = [  # (B, H, W, C, stride)
    (1, 2, 2, 8, 2), (1, 3, 3, 8, 2), (1, 2, 3, 8, 2), (2, 5, 4, 72, 2), (1, 7, 7, 144, 2), (2, 4, 5, 384, 2),
    (1, 9, 6, 96, 2), (1, 6, 9, 192, 2), (1, 11, 13, 576, 2), (1, 1, 1, 8, 1), (1, 2, 3, 96, 1), (1, 6, 9, 192, 1),
    (1, 3, 2, 576, 1), (2, 11, 10, 72, 1), (1, 8, 8, 144, 1), (1, 5, 7, 384, 1)]
REDUCE_CASES = [(1, 7, 13, 8), (2, 5, 9, 64), (1, 11, 3, 120), (1, 6, 7, 240), (3, 5, 5, 512), (1, 1, 1, 512),
                (1, 1, 1, 8)]
_CD = (1, 2, 5, 11, 12, 15, 16, 17, 31, 33, 64)
CDCM_CASES = sorted({(1, h, w) for h, w in zip(_CD, _CD)} | {(1, h, w) for h, w in zip(_CD, _CD[::-1])}
                    | {(3, 17, 33), (1, 131, 97), (1, 65, 48), (1, 32, 24), (1, 16, 12)})
SIDE_CASES = [(1, 1, 1), (1, 1, 5), (2, 2, 3), (1, 3, 2), (3, 7, 5), (1, 17, 13), (2, 33, 31)]
FUSE_CASES = [(1, 8, 8), (2, 9, 11), (2, 37, 45), (1, 67, 61), (2, 65, 64), (2, 131, 97), (1, 200, 9)]
UPSAMPLE_CASES = [(1, 1, 1), (1, 1, 5), (2, 4, 1), (1, 3, 7), (2, 16, 9), (1, 33, 32)]
MLSD_HEAD_CASES = [(1, 7, 9, 8), (2, 5, 3, 128), (1, 4, 4, 256), (2, 13, 11, 256)]
OP_HEAD_CASES = [  # (B, h, w, C, N, relu, out_c, out_off)
    (1, 5, 7, 128, 38, False, 57, 0), (2, 4, 3, 128, 19, True, 57, 38), (1, 6, 5, 136, 71, True, 90, 10),
    (1, 3, 3, 128, 71, False, 71, 0)]


def pool_input(B, H, W, C, integer, seed):
    """fp16 channel-last map: integers in [-3, 3] (many ties among the four inputs) or fp16 normals."""
    return (ints((B, H, W, C), -3, 3, seed) if integer else randn((B, H, W, C), seed)).half()


def dw_inputs(B, H, W, C, ks, integer, seed):
    """(x fp16 [B,H,W,C], w [C,1,ks,ks] fp32); channels 60.. zero-weighted as the network pads 60 channels to 64.
    Integer case: |x| <= 4, |w| <= 3, so every sum (<= 300) is exact."""
    if integer:
        x, w4 = ints((B, H, W, C), -4, 4, seed), ints((C, 1, ks, ks), -3, 3, seed + 1)
    else:
        x, w4 = randn((B, H, W, C), seed), randn((C, 1, ks, ks), seed + 1, 0.3)
    if C == 64:
        w4[60:] = 0
    return x.half(), w4.float()


def mlsd_dw_inputs(B, H, W, C, integer, seed):
    """(x, w4 [C,1,3,3], b): x >= 0 up to 10 (a ReLU output; min(x, 6) matters), a bias pushing outputs to both clamp
    ends.  Integer case: x integers, w multiples of 1/8 in [-1/4, 1/4], b multiples of 1/2: sums exact."""
    if integer:
        x = ints((B, H, W, C), 0, 10, seed)
        w4, b = ints((C, 1, 3, 3), -2, 2, seed + 1, 0.125), ints((C,), -6, 6, seed + 2, 0.5)
    else:
        x = rand((B, H, W, C), seed, 0.0, 10.0)
        w4, b = randn((C, 1, 3, 3), seed + 1, 0.3), randn((C,), seed + 2, 2.0)
    return x.half(), w4.float(), b.float()


def reduce_inputs(B, h, w, C, integer, seed):
    """(x fp16 with negatives (the ReLU matters), w [C, 24], b [24]).  Integer: |x| <= 2, |w| <= 1, |b| <= 8."""
    if integer:
        return (ints((B, h, w, C), -2, 2, seed).half(), ints((C, D), -1, 1, seed + 1).float(),
                ints((D,), -8, 8, seed + 2).float())
    return randn((B, h, w, C), seed).half(), randn((C, D), seed + 1, 0.2).float(), randn((D,), seed + 2).float()


def cdcm_inputs(B, h, w, integer, seed):
    """(m fp16 [B,h,w,24], Ws [4,24,24,3,3] fp16 values).  Integer: m, W in [-2, 2], |u| <= 864 * 4 = 3456, every
    partial sum an integer below 2^24."""
    if integer:
        return ints((B, h, w, D), -2, 2, seed).half(), ints((4, D, D, 3, 3), -2, 2, seed + 1).half().float()
    return randn((B, h, w, D), seed).half(), randn((4, D, D, 3, 3), seed + 1, 0.1).half().float()


def side_inputs(B, h, w, seed):
    return randn((B, h, w, D), seed, 2.0).float(), side_params(seed + 10)


def fuse_inputs(B, H, W, seed):
    """Four side maps [B,h_k,w_k] at the network's sizes (different per image) and the classifier [w0..w3, b]."""
    sides = [randn((B, h, w), seed + k, 2.0).float() for k, (h, w) in enumerate(fuse_sizes(H, W))]
    return sides, (randn((5,), seed + 9) * torch.tensor([1.0, 1.0, 1.0, 1.0, 0.5], dtype=torch.float64)).float()


def upsample_input(B, h, w, C, seed):
    return randn((B, h, w, C), seed).half()


def head_inputs(B, h, w, C, N, integer, seed):
    """(x fp16, w [N, C], b [N]).  Integer: |x| <= 3, |w| <= 2, |b| <= 8 (exact)."""
    if integer:
        return (ints((B, h, w, C), -3, 3, seed).half(), ints((N, C), -2, 2, seed + 1).float(),
                ints((N,), -8, 8, seed + 2).float())
    return randn((B, h, w, C), seed).half(), randn((N, C), seed + 1, 0.1).float(), randn((N,), seed + 2).float()


# ------------------------------------------------------------------------------------------------- checks
# Each check builds a case's inputs, calls `run` (the kernel's wrapper, or an emulation standing in for it) and
# compares with the reference.  It returns (ok, worst): for an integer case worst is the number of values that differ
# from the exact result (+0 and -0 count as equal: the sign of an exact zero is not part of the arithmetic), for a
# random case the largest error as a fraction of the bound.  Data movement is compared bit for bit.
INF = float("inf")


def bit_mismatches(out: torch.Tensor, ref: torch.Tensor) -> int:
    out = out.cpu()
    if tuple(out.shape) != tuple(ref.shape) or out.dtype != ref.dtype:
        return max(out.numel(), ref.numel(), 1)
    w = {2: torch.int16, 4: torch.int32, 1: torch.uint8}[out.element_size()]
    return int((out.contiguous().view(w) != ref.contiguous().view(w)).sum())


def _verdict(out, ref, bound, integer):
    out = out.cpu()
    if tuple(out.shape) != tuple(ref.shape):
        return False, INF
    if integer:
        n = mismatches(out, ref)
        return n == 0, float(n)
    r = err_ratio(out, ref, bound)
    return r <= 1.0, r


def check_quant(run_roundtrip, run_hed, run_mlsd, dtype, mutant_ref=None):
    """All three quantiser entry points on the dtype's input set -> (ok, bit mismatches)."""
    vals = quant_inputs_f16() if dtype == torch.float16 else quant_inputs_f32().to(dtype)
    n = bit_mismatches(run_roundtrip(vals), to_u8_ref(vals).float() / 255)
    img, _ = as_image(vals)
    for norm, scale in ((HED_NORM, HED_SCALE), ((0.0, 0.0, 0.0), 1.0)):
        for cpad in (3, 16):
            n += bit_mismatches(run_hed(img, norm, scale, cpad), hed_input_ref(img, norm, scale, cpad))
    n += bit_mismatches(run_mlsd(img), mlsd_input_ref(img))
    return n == 0, float(n)


def check_pool(run, case, integer, seed):
    x = pool_input(*case, integer, seed)
    n = bit_mismatches(run(x), pool_ref(x))
    return n == 0, float(n)


def check_im2col(run, case, seed):
    x = pool_input(*case, False, seed)
    n = bit_mismatches(run(x), im2col7_ref(x))
    return n == 0, float(n)


def check_dw(run, case, integer, seed):
    B, H, W, C, ks, pool = case
    x, w4 = dw_inputs(B, H, W, C, ks, integer, seed)
    res = run(x, dw_weights(w4), pool)
    out, pooled = res if pool else (res, None)
    ref, bound, pref = pidinet_dw_ref(x, w4, pool)
    ok, worst = _verdict(out, ref, bound, integer)
    if pool:
        ok = ok and bit_mismatches(pooled, pref.half()) == 0
    if ok and C == 64:                             # zero-weighted pad channels are exactly 0
        ok = bool((out.cpu()[..., 60:].float() == 0).all())
    return ok, worst


def check_mlsd_dw(run, case, integer, seed):
    B, H, W, C, stride = case
    x, w4, b = mlsd_dw_inputs(B, H, W, C, integer, seed)
    out = run(x, dw_weights(w4), b, stride)
    return _verdict(out, *mlsd_dw_ref(x, w4, b, stride), integer)


def check_reduce(run, case, integer, seed):
    x, w, b = reduce_inputs(*case, integer, seed)
    return _verdict(run(x, w, b), *reduce_ref(x, w, b), integer)


def check_cdcm(run, case, integer, seed, pack=None):
    from pfd_b200.pidinet import pack_cdcm
    m, Ws = cdcm_inputs(*case, integer, seed)
    wpk = (pack or pack_cdcm)(list(Ws))
    return _verdict(run(m, wpk), *cdcm_ref(m, Ws), integer)


def check_side(run, case, seed):
    u, prm = side_inputs(*case, seed)
    return _verdict(run(u, prm), *side_ref(u, prm), False)


def check_fuse(run, case, seed):
    """(ok, pixels near an integer): levels exact away from integers, near-integer pixels at most 1 in 10^4."""
    B, H, W = case
    sides, cls = fuse_inputs(B, H, W, seed)
    levels, pre = fuse_ref(sides, cls, H, W)
    bad, near, exact = fuse_check(run(sides, cls, H, W), levels, pre)
    return bad == 0 and exact and near <= B * H * W // 10000, float(near)


def check_upsample(run, case, seed, C=64):
    """Into the [..., 64:] half of a 128-channel buffer filled with a sentinel: the other half keeps its bits; also
    within one fp16 ulp of F.interpolate on fp32."""
    B, h, w = case
    x = upsample_input(B, h, w, C, seed)
    buf = torch.full((B, 2 * h, 2 * w, 2 * C), -1234.0, dtype=torch.float16)
    buf = run(x, buf)
    ref, bound = upsample_ref(x)
    ok, worst = _verdict(buf[..., C:], ref, bound, False)
    ok = ok and bit_mismatches(buf[..., :C], torch.full((B, 2 * h, 2 * w, C), -1234.0, dtype=torch.float16)) == 0
    # one fp16 ulp, plus the fp32 evaluation error of both sides where neighbours of opposite sign cancel
    it = nhwc(F.interpolate(nchw(x.float()), scale_factor=2, mode="bilinear", align_corners=True)).double()
    tol = ulp16(it) + 8 * U32 * upsample_ref(x.abs())[0]
    ok = ok and bool(((buf[..., C:].cpu().double() - it).abs() <= tol).all())
    return ok, worst


def check_mlsd_head(run, case, integer, seed):
    x, w, b = head_inputs(*case, 5, integer, seed)
    return _verdict(run(x, w, b), *head_ref(x, w, b, False), integer)


def check_op_head(run, case, integer, seed):
    """Written at out_off into a wider planar buffer filled with a sentinel: the other channels keep their bits."""
    B, h, w, C, N, relu, out_c, off = case
    x, wt, b = head_inputs(B, h, w, C, N, integer, seed)
    buf = torch.full((B, out_c, h, w), -777.0)
    buf = run(x, wt, b, relu, buf, off).cpu()
    ok, worst = _verdict(buf[:, off:off + N], *head_ref(x, wt, b, relu), integer)
    keep = torch.cat([buf[:, :off], buf[:, off + N:]], 1)
    return ok and bit_mismatches(keep, torch.full_like(keep, -777.0)) == 0, worst


# ------------------------------------------------------------------------------------------------- emulated kernels
def model_runners(mutant=None):
    """The emulations with the `run` signatures of the checks (the GPU test passes the wrappers instead)."""
    def up(x, buf):
        buf = buf.clone()
        buf[..., buf.shape[-1] // 2:] = upsample_model(x, mutant)
        return buf

    def op_head(x, w, b, relu, buf, off):
        buf = buf.clone()
        buf[:, off:off + w.shape[0]] = head_model(x, w, b, relu, mutant)
        return buf

    return {
        "roundtrip": lambda v: to_u8_model(v, mutant).float() / 255,
        "hed_input": lambda img, norm, scale, cpad: _hed_input_model(img, norm, scale, cpad, mutant),
        "mlsd_input": lambda img: _mlsd_input_model(img, mutant),
        "pool": lambda x: pool_model(x, mutant),
        "im2col": im2col7_ref,
        "dw": lambda x, wt, pool: pidinet_dw_model(x, wt, pool, mutant),
        "mlsd_dw": lambda x, wt, b, s: mlsd_dw_model(x, wt, b, s, mutant),
        "reduce": reduce_model,
        "cdcm": lambda m, wpk: cdcm_model(m, wpk, mutant),
        "side": lambda u, prm: side_model(u, prm, mutant),
        "fuse": lambda sides, cls, H, W: _fuse_out(*fuse_model(sides, cls, H, W, mutant)),
        "upsample": up,
        "mlsd_head": lambda x, w, b: head_model(x, w, b, False),
        "op_head": op_head,
    }


def _hed_input_model(img, norm, scale, cpad, mutant):
    u = to_u8_model(img, mutant).float().numpy()
    v = ((u - np.asarray(norm, F32).reshape(1, 3, 1, 1)).astype(F32) * F32(scale)).astype(F32).astype(np.float16)
    B, _, H, W = img.shape
    out = np.zeros((B, H, W, cpad), np.float16)
    out[..., :3] = v.transpose(0, 2, 3, 1)
    return torch.from_numpy(out)


def _mlsd_input_model(img, mutant):
    u = to_u8_model(img, mutant).float().numpy()
    B, _, H, W = img.shape
    out = np.zeros((B, H, W, 16), np.float16)
    out[..., :3] = (u - F32(127.5)).transpose(0, 2, 3, 1)
    out[..., 3] = -126.5
    return torch.from_numpy(out)


def _fuse_out(levels, pre):
    v = levels.float() / 255
    return v[:, None].expand(-1, 3, -1, -1).contiguous()
