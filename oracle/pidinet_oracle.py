"""CPU / fp32 restatement of the PiDiNet soft-edge step behind ControlNet.preprocess(type='scribble') (the default
method 'pidinet').  TEST INFRASTRUCTURE — only tests/ and tools/ may import this module.

Reference path: lib/model_zoo/controlnet.py:465-472 (tensor -> ToPILImage -> apply_pidinet -> make_scribble) and
lib/model_zoo/controlnet_annotator/pidinet/__init__.py:67-96 around the network pidinet() of pidinet/model.py:441-666
(config 'carv4', 60 channels, dil=24, sa=True), written here from its description:
  * input: the uint8 RGB image flipped to BGR, / 255 in float32;
  * init block: a 3x3 pixel-difference conv 3 -> 60 (no bias), then four stages of four blocks with 60 / 120 / 240 /
    240 channels.  A block is depthwise PDC conv -> ReLU -> 1x1 conv (no bias) + x; the first block of stages 2-4 max-pools
    2x2 first and replaces `+ x` by a 1x1 shortcut conv with bias;
  * the 16 PDC layers follow 'carv4': layer i is cd, ad, rd, cv for i % 4 = 0, 1, 2, 3 (layer 0 is the init block);
    each is a plain convolution once its weight is converted (`convert_pdc`);
  * per stage: CDCM (ReLU, 1x1 to 24 with bias, sum of four 3x3 convs 24 -> 24 with dilation 5 / 7 / 9 / 11 and
    matching zero padding, no bias), CSAM (u * sigmoid(conv3x3(conv1x1_4(relu(u)) + b), padding 1, no bias)) and
    MapReduce (1x1 to one channel with bias): the pre-sigmoid side map e_k;
  * each e_k upsampled to H x W with F.interpolate(bilinear, align_corners=False) (restated in numpy by
    `resize_bilinear`, pinned bit for bit against torch by tests/test_pidinet_cpu.py), the classifier 1x1 conv 4 -> 1
    with bias, sigmoid, then (edge * 255).clip(0, 255).astype(uint8).
"""
import numpy as np
import torch
import torch.nn.functional as F

C0 = 60                                  # stage-1 width
DIL = 24                                 # CDCM / CSAM / MapReduce width
DILATIONS = (5, 7, 9, 11)
STAGE_CH = (C0, 2 * C0, 4 * C0, 4 * C0)
PDC_ORDER = ("cd", "ad", "rd", "cv")     # 'carv4': layer i uses PDC_ORDER[i % 4]
# Synthetic-weight contrast: with plain name-seeded weights the output levels sit in a narrow band around 128 (115..159
# on a 256^2 test image), which leaves the level and scribble checks nearly vacuous.  The classifier weights are
# multiplied by this gain in `synth_state_dict`; the same image then spans levels 18..252.
CLASSIFIER_GAIN = 10.0
# ad: w - w[AD_PERM] (flattened 3x3, clockwise neighbour); rd: 5x5 ring positions that take +w[1:] / -w[1:]
AD_PERM = (3, 0, 1, 6, 4, 2, 7, 8, 5)
RD_OUTER = (0, 2, 4, 10, 14, 20, 22, 24)
RD_INNER = (6, 7, 8, 11, 13, 16, 17, 18)


def block_names():
    """[(name, stage, layer index, cin, cout, stride)] of the 15 PDC blocks after the init block."""
    out = []
    layer = 1
    for s in range(4):
        cin = STAGE_CH[s - 1] if s else C0
        cout = STAGE_CH[s]
        for j in range(4):
            if s == 0 and j == 3:
                break
            name = f"block{s + 1}_{j + 1}"
            first = j == 0 and s > 0
            out.append((name, s, layer, cin if first else cout, cout, 2 if first else 1))
            layer += 1
    return out


def state_dict_shapes():
    """{key: shape} of the annotator's state dict (table5_pidinet.pth without the 'module.' prefix), in module order."""
    out = {"init_block.weight": (C0, 3, 3, 3)}
    for name, _, _, cin, cout, stride in block_names():
        if stride > 1:
            out[f"{name}.shortcut.weight"] = (cout, cin, 1, 1)
            out[f"{name}.shortcut.bias"] = (cout,)
        out[f"{name}.conv1.weight"] = (cin, 1, 3, 3)
        out[f"{name}.conv2.weight"] = (cout, cin, 1, 1)
    for i in range(4):
        out[f"conv_reduces.{i}.conv.weight"] = (1, DIL, 1, 1)
        out[f"conv_reduces.{i}.conv.bias"] = (1,)
    for i in range(4):
        out[f"attentions.{i}.conv1.weight"] = (4, DIL, 1, 1)
        out[f"attentions.{i}.conv1.bias"] = (4,)
        out[f"attentions.{i}.conv2.weight"] = (1, 4, 3, 3)
    for i in range(4):
        out[f"dilations.{i}.conv1.weight"] = (DIL, STAGE_CH[i], 1, 1)
        out[f"dilations.{i}.conv1.bias"] = (DIL,)
        for j in range(4):
            out[f"dilations.{i}.conv2_{j + 1}.weight"] = (DIL, DIL, 3, 3)
    out["classifier.weight"] = (1, 4, 1, 1)
    out["classifier.bias"] = (1,)
    return out


def synth_state_dict(seed=0):
    """Name-seeded synthetic weights (pfd_b200/weights.py synth_tensor), classifier.weight times CLASSIFIER_GAIN."""
    from pfd_b200.weights import synth_tensor
    sd = {k: synth_tensor(k, s, seed) for k, s in state_dict_shapes().items()}
    sd["classifier.weight"] = sd["classifier.weight"] * CLASSIFIER_GAIN
    return sd


def fill_synthetic(module, seed=0):
    """Load the synthetic weights into a module with the annotator's keys (ours or the reference's), strict=True."""
    sd = synth_state_dict(seed)
    dev = next(module.parameters()).device
    module.load_state_dict({k: v.to(dev) for k, v in sd.items()}, strict=True)
    return module


def convert_pdc(op, w):
    """Pixel-difference weights [C, 1, 3, 3] -> plain conv weights ([C,1,3,3], or [C,1,5,5] for 'rd' with padding 2)."""
    c = w.shape[0]
    f = w.reshape(c, -1, 9)
    if op == "cv":
        return w.clone()
    if op == "cd":                       # conv(x, w) - conv1x1(x, sum w) == conv(x, w with centre -= sum)
        out = f.clone()
        out[:, :, 4] = out[:, :, 4] - f.sum(-1)
        return out.reshape(w.shape)
    if op == "ad":
        return (f - f[:, :, list(AD_PERM)]).reshape(w.shape)
    if op == "rd":
        out = torch.zeros((c, f.shape[1], 25), dtype=w.dtype)
        out[:, :, list(RD_OUTER)] = f[:, :, 1:]
        out[:, :, list(RD_INNER)] = -f[:, :, 1:]
        return out.reshape(c, f.shape[1], 5, 5)
    raise ValueError(op)


def _shift(x, dy, dx):
    """x[..., y + dy, x + dx], zero outside the image."""
    H, W = x.shape[-2:]
    p = F.pad(x, (2, 2, 2, 2))
    return p[..., 2 + dy:2 + dy + H, 2 + dx:2 + dx + W]


def pdc_reference_form(op, x, w):
    """A depthwise pixel-difference convolution (x [N,C,H,W], w [C,1,3,3]) as a weighted sum of pixel differences,
    with no weight conversion, for pinning `convert_pdc`:
      cv  sum_j w_j x(p_j)                       cd  sum_j w_j (x(p_j) - x(centre))
      ad  sum_j w_j (x(p_j) - x(p_q(j))), q the inverse of AD_PERM
      rd  sum_{i=1..8} w_i (x(RD_OUTER[i-1]) - x(RD_INNER[i-1])) on the 5x5 window (w_0 is unused)."""
    c = w.shape[0]
    f = w.reshape(1, c, 9, 1, 1)
    off3 = [(j // 3 - 1, j % 3 - 1) for j in range(9)]
    off5 = lambda p: (p // 5 - 2, p % 5 - 2)                                  # noqa: E731
    if op == "cv":
        return sum(f[:, :, j] * _shift(x, *off3[j]) for j in range(9))
    if op == "cd":
        return sum(f[:, :, j] * (_shift(x, *off3[j]) - x) for j in range(9))
    if op == "ad":
        q = [AD_PERM.index(j) for j in range(9)]
        return sum(f[:, :, j] * (_shift(x, *off3[j]) - _shift(x, *off3[q[j]])) for j in range(9))
    if op == "rd":
        return sum(f[:, :, i] * (_shift(x, *off5(RD_OUTER[i - 1])) - _shift(x, *off5(RD_INNER[i - 1])))
                   for i in range(1, 9))
    raise ValueError(op)


def pdc_of_layer(i):
    return PDC_ORDER[i % 4]


def network_sides(sd, img_u8, device="cpu", return_acts=False):
    """The four pre-sigmoid side maps e_k (float32 numpy [h_k, w_k]) of the network on one HxWx3 uint8 RGB image."""
    with torch.no_grad():
        p = {k: v.to(device=device, dtype=torch.float32) for k, v in sd.items()}
        x = torch.from_numpy(np.ascontiguousarray(img_u8[:, :, ::-1]).astype(np.float32)).to(device)
        x = (x / 255.0).permute(2, 0, 1)[None]
        h = F.conv2d(x, convert_pdc("cd", p["init_block.weight"].cpu()).to(device), padding=1)
        stage_out, acts = [], []
        for name, s, layer, cin, cout, stride in block_names():
            if stride > 1:
                stage_out.append(h)
                h = F.max_pool2d(h, 2, 2)
            op = pdc_of_layer(layer)
            wd = convert_pdc(op, p[f"{name}.conv1.weight"].cpu()).to(device)
            y = F.relu(F.conv2d(h, wd, padding=wd.shape[-1] // 2, groups=cin))
            y = F.conv2d(y, p[f"{name}.conv2.weight"])
            h = y + (F.conv2d(h, p[f"{name}.shortcut.weight"], p[f"{name}.shortcut.bias"]) if stride > 1 else h)
            acts.append(float(h.abs().max()))
        stage_out.append(h)
        sides = []
        for i, xs in enumerate(stage_out):
            m = F.conv2d(F.relu(xs), p[f"dilations.{i}.conv1.weight"], p[f"dilations.{i}.conv1.bias"])
            u = sum(F.conv2d(m, p[f"dilations.{i}.conv2_{j + 1}.weight"], padding=d, dilation=d)
                    for j, d in enumerate(DILATIONS))
            a = F.conv2d(F.relu(u), p[f"attentions.{i}.conv1.weight"], p[f"attentions.{i}.conv1.bias"])
            a = torch.sigmoid(F.conv2d(a, p[f"attentions.{i}.conv2.weight"], padding=1))
            e = F.conv2d(u * a, p[f"conv_reduces.{i}.conv.weight"], p[f"conv_reduces.{i}.conv.bias"])
            sides.append(e[0, 0].cpu().numpy().astype(np.float32))
    return (sides, acts) if return_acts else sides


def _fma(a, b, c):
    """float32 fused multiply-add (the float64 product of two float32 values is exact)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _coords(dst, src):
    """PyTorch's bilinear source rule (align_corners=False, no scale factor): scale = float32(src / dst),
    pos = max(0, fma(d + 0.5, scale, -0.5)) in float32; index = floor, lambda = pos - index, the second index clamped
    at the edge."""
    scale = np.float32(src) / np.float32(dst)
    d = np.arange(dst, dtype=np.float32) + np.float32(0.5)
    pos = np.maximum(_fma(d, scale, np.float32(-0.5)), np.float32(0))
    i0 = pos.astype(np.int64)
    lam = (pos - i0.astype(np.float32)).astype(np.float32)
    return i0, np.minimum(i0 + 1, src - 1), lam


def _lerp(a0, a1, lam):
    """fma(a0, 1 - lam, a1 * lam) in float32."""
    return _fma(a0, np.float32(1) - lam, (a1 * lam).astype(np.float32))


def resize_bilinear(src, H, W):
    """F.interpolate(src[None, None], (H, W), mode='bilinear', align_corners=False)[0, 0] of a float32 [h, w] map, as
    PyTorch's CPU kernel computes it for H + W > 128 (its separable path): a pass along the width into float32, then one
    along the height, each skipped when that size does not change.  Bit-exact there (tests/test_pidinet_cpu.py); for
    smaller outputs PyTorch takes another path whose values differ by an ulp or so."""
    out = np.asarray(src, np.float32)
    h, w = out.shape
    if w != W:
        x0, x1, lx = _coords(W, w)
        out = _lerp(out[:, x0], out[:, x1], lx[None, :])
    if h != H:
        y0, y1, ly = _coords(H, h)
        out = _lerp(out[y0], out[y1], ly[:, None])
    return out


def fuse(sd, sides, H, W):
    """apply_pidinet after the side maps -> (uint8 [H, W] edge map, float64 pre-quantisation value edge * 255)."""
    cw = sd["classifier.weight"].reshape(4).double().numpy()
    cb = float(sd["classifier.bias"].reshape(1)[0])
    acc = np.full((H, W), cb, np.float64)
    for k, s in enumerate(sides):
        acc += cw[k] * resize_bilinear(s, H, W).astype(np.float64)
    edge = 1.0 / (1.0 + np.exp(-acc))
    pre = edge * 255.0
    return pre.clip(0, 255).astype(np.uint8), pre


def apply_pidinet(sd, img_u8, device="cpu"):
    """-> (uint8 edge map, pre-quantisation value, side maps)."""
    H, W = img_u8.shape[:2]
    sides = network_sides(sd, img_u8, device)
    u8, pre = fuse(sd, sides, H, W)
    return u8, pre, sides


def near_integer(pre, tol=1e-3):
    """Pixels whose pre-quantisation value lies within tol of an integer (their uint8 level may flip either way)."""
    return np.abs(pre - np.round(pre)) <= tol
