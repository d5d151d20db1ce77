"""CPU / fp32 restatement of the HED soft-edge step of ControlNet.preprocess.  TEST INFRASTRUCTURE — only tests/ and
tools/ may import this module.

Reference path: lib/model_zoo/controlnet.py:370-376 (tensor -> ToPILImage -> apply_hed -> ToTensor -> repeat(1,3,1,1)
-> float32) and lib/model_zoo/controlnet_annotator/hed/__init__.py:102-128, written here from its description:
  * network (ControlNetHED_Apache2): h = x - norm on the 0..255 uint8 image in float32; five blocks of 2/2/3/3/3
    3x3 convolutions (padding 1, each followed by ReLU) with 64/128/256/512/512 channels, a 2x2 stride-2 max-pool in
    front of blocks 2-5, and a 1x1 convolution to one channel (the side map) at the end of every block;
  * each side map resized to the image size with cv2.resize(INTER_LINEAR) (restated in numpy by `resize_linear`,
    pinned against cv2 by tests/test_hed_cpu.py), stacked, np.mean over the five maps in float32, a float64
    sigmoid, then (edge * 255).clip(0, 255).astype(uint8).
"""
import numpy as np
import torch
import torch.nn.functional as F

BLOCKS = [(3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3)]


def state_dict_shapes():
    """{key: shape} of the annotator's state dict (ControlNetHED.pth)."""
    out = {"norm": (1, 3, 1, 1)}
    for bi, (cin, cout, layers) in enumerate(BLOCKS):
        for li in range(layers):
            out[f"block{bi + 1}.convs.{li}.weight"] = (cout, cin if li == 0 else cout, 3, 3)
            out[f"block{bi + 1}.convs.{li}.bias"] = (cout,)
        out[f"block{bi + 1}.projection.weight"] = (1, cout, 1, 1)
        out[f"block{bi + 1}.projection.bias"] = (1,)
    return out


def synth_state_dict(seed=0):
    """Name-seeded synthetic weights (pfd_b200/weights.py synth_tensor) for every key of the annotator."""
    from pfd_b200.weights import synth_tensor
    return {k: synth_tensor(k, s, seed) for k, s in state_dict_shapes().items()}


def fill_synthetic(module, seed=0):
    """Load the synthetic weights into a module with the annotator's keys (ours or the reference's), strict=True."""
    sd = synth_state_dict(seed)
    dev = next(module.parameters()).device
    module.load_state_dict({k: v.to(dev) for k, v in sd.items()}, strict=True)
    return module


def hed_image(seed, H, W):
    """Deterministic smooth-plus-detail HxWx3 uint8 test image."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((1, 3, H, W), generator=g)
    x = 0.6 * F.avg_pool2d(x, 9, 1, 4, count_include_pad=False) + 0.4 * F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
    x = (x - x.min()) / (x.max() - x.min())
    return (x[0].permute(1, 2, 0) * 255).round().clamp(0, 255).to(torch.uint8).numpy()


def image_to_tensor(img_u8, dtype=torch.float32):
    """[1,3,H,W] tensor in [0,1] whose ToPILImage quantisation x.mul(255).byte() gives back img_u8 exactly."""
    x = (torch.from_numpy(img_u8.astype(np.float32)).permute(2, 0, 1)[None] + 0.5) / 255.0
    return x.to(dtype)


def to_pil_u8(x):
    """ToPILImage on a float [3,H,W] tensor: x.mul(255).byte() -> HxWx3 uint8 (rounded in x's dtype)."""
    return x.mul(255).byte().permute(1, 2, 0).contiguous().cpu().numpy()


def network_sides(sd, img_u8, device="cpu"):
    """The five side maps (float32 numpy [h_k, w_k]) of the network on one HxWx3 uint8 image, in fp32."""
    with torch.no_grad():
        p = {k: v.to(device=device, dtype=torch.float32) for k, v in sd.items()}
        h = torch.from_numpy(img_u8.astype(np.float32)).to(device).permute(2, 0, 1)[None] - p["norm"]
        sides = []
        for bi, (_, _, layers) in enumerate(BLOCKS):
            if bi > 0:
                h = F.max_pool2d(h, 2, 2)
            for li in range(layers):
                h = F.relu(F.conv2d(h, p[f"block{bi + 1}.convs.{li}.weight"], p[f"block{bi + 1}.convs.{li}.bias"],
                                    padding=1))
            s = F.conv2d(h, p[f"block{bi + 1}.projection.weight"], p[f"block{bi + 1}.projection.bias"])
            sides.append(s[0, 0].cpu().numpy().astype(np.float32))
    return sides


def _coords(dst, src):
    """Source index / float32 fraction of cv2's INTER_LINEAR rule: (d + 0.5) * (1 / (dst / src)) - 0.5 in double."""
    f = (np.arange(dst) + 0.5) * (1.0 / (dst / src)) - 0.5
    i = np.floor(f)
    return i.astype(np.int64), (f - i).astype(np.float32)


def resize_linear(src, H, W):
    """cv2.resize(src, (W, H), interpolation=cv2.INTER_LINEAR) of a float32 [h, w] map, for upscaling and equal sizes:
    columns clamped at the borders with a zero fraction, rows clipped to the image; horizontal pass, then vertical."""
    src = np.asarray(src, np.float32)
    h, w = src.shape
    if (h, w) == (H, W):
        return src.copy()
    one = np.float32(1)
    sx, fx = _coords(W, w)
    lo, hi = sx < 0, sx >= w - 1
    sx[lo], fx[lo] = 0, 0
    sx[hi], fx[hi] = w - 1, 0
    sx1 = np.minimum(sx + 1, w - 1)
    hor = src[:, sx] * (one - fx) + src[:, sx1] * fx
    sy, fy = _coords(H, h)
    r0, r1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    return hor[r0] * (one - fy)[:, None] + hor[r1] * fy[:, None]


def fuse(sides, H, W):
    """apply_hed after the network: -> (uint8 [H, W] edge map, float64 pre-quantisation value edge * 255)."""
    acc = None
    for s in sides:                                     # np.mean over a float32 axis of 5: sequential sum, then / 5
        r = resize_linear(s, H, W)
        acc = r if acc is None else acc + r
    m = acc / np.float32(len(sides))
    edge = 1.0 / (1.0 + np.exp(-m.astype(np.float64)))
    pre = edge * 255.0
    return pre.clip(0, 255).astype(np.uint8), pre


def apply_hed(sd, img_u8, device="cpu"):
    """-> (uint8 edge map, pre-quantisation value, side maps)."""
    H, W = img_u8.shape[:2]
    sides = network_sides(sd, img_u8, device)
    u8, pre = fuse(sides, H, W)
    return u8, pre, sides


def near_integer(pre, tol=1e-3):
    """Pixels whose pre-quantisation value lies within tol of an integer (their uint8 level may flip either way)."""
    return np.abs(pre - np.round(pre)) <= tol
