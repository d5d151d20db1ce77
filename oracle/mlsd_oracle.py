"""CPU / fp32 restatement of the M-LSD line annotator behind ControlNet.preprocess(type='mlsd' / 'mlsd_v11p').
TEST INFRASTRUCTURE - only tests/ and tools/ may import this module.  It imports no cv2.

Reference path: lib/model_zoo/controlnet.py:378-386 (tensor -> ToPILImage -> apply_mlsd per image -> ToTensor ->
repeat) and lib/model_zoo/controlnet_annotator/mlsd (__init__.py:56-81, utils.py:18-88) around the network
MobileV2_MLSD_Large (models/mbv2_mlsd_large.py), written here from its description:
  * input: concat(rgb_u8, ones) as 4 channels, / 127.5 - 1 in float32, at the image's own size (pred_lines is called
    with input_shape = the image size, so its INTER_AREA resize is the identity and the ratios are 1);
  * MobileNetV2 trunk features[0..13]: a 3x3 stride-2 stem 4 -> 32, then inverted residuals (t, c, n, s) =
    (1,16,1,1), (6,24,2,2), (6,32,3,2), (6,64,4,2), (6,96,3,1).  Every conv has BN (eval, eps 1e-5) and ReLU6 except
    the linear projection; stride-2 convs pad (0,1,0,1) with zeros, then use padding 0 (TFLite);
  * decoder: BlockTypeA (1x1 + BN + ReLU on both inputs, bilinear x2 with align_corners=True of the second unless
    block15, concat), BlockTypeB (3x3 + BN + ReLU, + x, 3x3 to 64 + BN + ReLU), BlockTypeC (dilation-5 3x3 + BN + ReLU,
    3x3 + BN + ReLU, 1x1 to 16), channels 7..11 kept: centre logit and the (start, end) displacements;
  * decode: sigmoid, 3x3 max-pool NMS, top-200 (torch.topk), score > thr_v and |start - end| > thr_d (float32, numpy
    promotes the Python thresholds to float32), endpoints int(2 * (x + d)) in float64;
  * cv2.line(..., 255, thickness 1, LINE_8) per segment: OpenCV's clipLine, then its LineIterator (8-connected,
    left to right), restated in `draw_line`.
Any exception inside the reference's pred_lines leaves a blank map; `size_supported` says when the shapes raise.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

TOPK = 200
BN_EPS = 1e-5
# (expand ratio t, output channels c, repeats n, first stride s) of the trunk (mbv2_mlsd_large.py:173-182)
TRUNK = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1))
FPN = (1, 3, 6, 10, 13)                  # features whose outputs c1..c5 feed the decoder
# (name, in_c1, in_c2, upscale) of the BlockTypeA blocks; each is followed by a BlockTypeB(128, 64)
DECODER = (("block15", 64, 96, False), ("block17", 32, 64, True), ("block19", 24, 64, True),
           ("block21", 16, 64, True))
KEEP = (7, 12)                           # output channels read by the decode: centre, start x, y, end x, y
# Synthetic-weight contrast.  With name-seeded weights and random BN statistics the centre logits and displacements
# are small (the centre logits vary by ~0.03, displacements by ~0.15 map px); `synth_state_dict` scales
# block23.conv3's row 7 (centre; its bias then moves by CENTRE_SHIFT) and rows 8..11 (displacements) by these gains,
# so the test images have peaks on both sides of thr_v, more than 200 above it on the larger images, and segments
# tens of pixels long that leave the image.
CENTRE_GAIN = 40.0
CENTRE_SHIFT = 6.0
DISP_GAIN = 120.0


def _bn_keys(prefix, c):
    return {f"{prefix}.weight": (c,), f"{prefix}.bias": (c,), f"{prefix}.running_mean": (c,),
            f"{prefix}.running_var": (c,), f"{prefix}.num_batches_tracked": ()}


def trunk_layers():
    """[(feature index, inp, hidden, oup, stride, residual)] of the inverted residuals features[1..13]."""
    out, inp, i = [], 32, 1
    for t, c, n, s in TRUNK:
        for j in range(n):
            stride = s if j == 0 else 1
            out.append((i, inp, int(round(inp * t)), c, stride, stride == 1 and inp == c))
            inp, i = c, i + 1
    return out


def state_dict_shapes():
    """{key: shape} of MobileV2_MLSD_Large's state dict (mlsd_large_512_fp32.pth), in module order."""
    out = {"backbone.features.0.0.weight": (32, 4, 3, 3)}
    out.update(_bn_keys("backbone.features.0.1", 32))
    for i, inp, hid, oup, _, _ in trunk_layers():
        p = f"backbone.features.{i}.conv"
        j = 0
        if hid != inp:
            out[f"{p}.0.0.weight"] = (hid, inp, 1, 1)
            out.update(_bn_keys(f"{p}.0.1", hid))
            j = 1
        out[f"{p}.{j}.0.weight"] = (hid, 1, 3, 3)
        out.update(_bn_keys(f"{p}.{j}.1", hid))
        out[f"{p}.{j + 1}.weight"] = (oup, hid, 1, 1)
        out.update(_bn_keys(f"{p}.{j + 2}", oup))
    for k, (name, c1, c2, _) in enumerate(DECODER):
        out[f"{name}.conv1.0.weight"] = (64, c2, 1, 1)
        out[f"{name}.conv1.0.bias"] = (64,)
        out.update(_bn_keys(f"{name}.conv1.1", 64))
        out[f"{name}.conv2.0.weight"] = (64, c1, 1, 1)
        out[f"{name}.conv2.0.bias"] = (64,)
        out.update(_bn_keys(f"{name}.conv2.1", 64))
        b = f"block{16 + 2 * k}"
        for conv, cout in (("conv1", 128), ("conv2", 64)):
            out[f"{b}.{conv}.0.weight"] = (cout, 128, 3, 3)
            out[f"{b}.{conv}.0.bias"] = (cout,)
            out.update(_bn_keys(f"{b}.{conv}.1", cout))
    for conv in ("conv1", "conv2"):
        out[f"block23.{conv}.0.weight"] = (64, 64, 3, 3)
        out[f"block23.{conv}.0.bias"] = (64,)
        out.update(_bn_keys(f"block23.{conv}.1", 64))
    out["block23.conv3.weight"] = (16, 64, 1, 1)
    out["block23.conv3.bias"] = (16,)
    return out


def synth_state_dict(seed=0):
    """Name-seeded synthetic weights (pfd_b200/weights.py synth_tensor) with random BN statistics (running_var in
    [0.5, 1.5), running_mean twice the name-seeded bias) and the output gains CENTRE_GAIN / DISP_GAIN."""
    from pfd_b200.weights import synth_tensor
    sd = {}
    for k, s in state_dict_shapes().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(s, generator=torch.Generator().manual_seed(len(k) * 7919 + seed))
        elif k.endswith("running_mean"):
            sd[k] = 2.0 * synth_tensor(k, s, seed)
        else:
            sd[k] = synth_tensor(k, s, seed)
    w, b = sd["block23.conv3.weight"].clone(), sd["block23.conv3.bias"].clone()
    w[7] *= CENTRE_GAIN
    b[7] = b[7] * CENTRE_GAIN + CENTRE_SHIFT
    w[8:12] *= DISP_GAIN
    sd["block23.conv3.weight"], sd["block23.conv3.bias"] = w, b
    return sd


def fill_synthetic(module, seed=0):
    """Load the synthetic weights into a module with the annotator's keys (ours or the reference's), strict=True."""
    sd = synth_state_dict(seed)
    dev = next(module.parameters()).device
    module.load_state_dict({k: v.to(dev) for k, v in sd.items()}, strict=True)
    return module


def fold_bn(sd, conv, bn):
    """Conv weight / bias with the eval-mode BN folded in (float64): w * g / sqrt(v + eps), (b - m) * g / sqrt + beta."""
    w = sd[conv + ".weight"].double()
    b = sd[conv + ".bias"].double() if conv + ".bias" in sd else torch.zeros(w.shape[0], dtype=torch.float64)
    g = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + BN_EPS)
    return w * g.reshape(-1, 1, 1, 1), (b - sd[bn + ".running_mean"].double()) * g + sd[bn + ".bias"].double()


def size_supported(H, W):
    """True when the reference's pred_lines runs on an H x W image: the decoder's concats need floor(H/2) and
    floor(W/2) to be multiples of 8 (the trunk halves sizes with floor), and torch.topk needs 200 map cells."""
    h, w = H // 2, W // 2
    return h % 8 == 0 and w % 8 == 0 and h > 0 and w > 0 and h * w >= TOPK


def network(sd, img_u8, device="cpu"):
    """Channels 7..11 of the network output (float32 numpy [5, H/2, W/2]) on one HxWx3 uint8 RGB image."""
    with torch.no_grad():
        p = {k: v.to(device=device, dtype=torch.float32) for k, v in sd.items() if v.is_floating_point()}
        H, W = img_u8.shape[:2]
        x = torch.from_numpy(np.ascontiguousarray(img_u8)).to(device).float().permute(2, 0, 1)[None]
        x = torch.cat([x, torch.ones((1, 1, H, W), device=device)], 1) / 127.5 - 1.0

        def cbr(x, conv, bn, stride=1, groups=1, act="relu6", pad=None):
            if stride == 2:
                x, pad = F.pad(x, (0, 1, 0, 1)), 0
            w = p[conv + ".weight"]
            k = w.shape[-1]
            x = F.conv2d(x, w, p.get(conv + ".bias"), stride, (k - 1) // 2 if pad is None else pad, groups=groups)
            if bn is not None:
                x = F.batch_norm(x, p[bn + ".running_mean"], p[bn + ".running_var"], p[bn + ".weight"],
                                 p[bn + ".bias"], False, 0.0, BN_EPS)
            return {"relu6": F.relu6, "relu": F.relu, None: lambda t: t}[act](x)

        feats = []
        x = cbr(x, "backbone.features.0.0", "backbone.features.0.1", stride=2)
        for i, inp, hid, oup, stride, res in trunk_layers():
            pre = f"backbone.features.{i}.conv"
            h, j = x, 0
            if hid != inp:
                h, j = cbr(h, f"{pre}.0.0", f"{pre}.0.1"), 1
            h = cbr(h, f"{pre}.{j}.0", f"{pre}.{j}.1", stride=stride, groups=hid)
            h = cbr(h, f"{pre}.{j + 1}", f"{pre}.{j + 2}", act=None)
            x = x + h if res else h
            if i in FPN:
                feats.append(x)
        c1, c2, c3, c4, c5 = feats
        x = c5
        for k, (name, _, _, up) in enumerate(DECODER):
            b = cbr(x, f"{name}.conv1.0", f"{name}.conv1.1", act="relu")
            a = cbr((c4, c3, c2, c1)[k], f"{name}.conv2.0", f"{name}.conv2.1", act="relu")
            if up:
                b = F.interpolate(b, scale_factor=2.0, mode="bilinear", align_corners=True)
            x = torch.cat((a, b), 1)
            blk = f"block{16 + 2 * k}"
            x = cbr(x, f"{blk}.conv1.0", f"{blk}.conv1.1", act="relu") + x
            x = cbr(x, f"{blk}.conv2.0", f"{blk}.conv2.1", act="relu")
        x = F.conv2d(x, p["block23.conv1.0.weight"], p["block23.conv1.0.bias"], padding=5, dilation=5)
        x = F.relu(F.batch_norm(x, p["block23.conv1.1.running_mean"], p["block23.conv1.1.running_var"],
                                p["block23.conv1.1.weight"], p["block23.conv1.1.bias"], False, 0.0, BN_EPS))
        x = cbr(x, "block23.conv2.0", "block23.conv2.1", act="relu")
        x = F.conv2d(x, p["block23.conv3.weight"][KEEP[0]:KEEP[1]], p["block23.conv3.bias"][KEEP[0]:KEEP[1]])
        return x[0].cpu().numpy().astype(np.float32)


def heat_map(centre):
    """sigmoid, then the 3x3 max-pool NMS of deccode_output_score_and_ptss: float32 [h, w] with 0 off the peaks."""
    heat = torch.sigmoid(torch.from_numpy(np.asarray(centre, np.float32)))[None]
    hmax = F.max_pool2d(heat, 3, stride=1, padding=1)
    return (heat * (hmax == heat).float())[0].numpy()


def decode(maps, thr_v=0.1, thr_d=0.1):
    """pred_lines after the network, for one image's [5, h, w] float32 map -> int64 [n, 4] segments
    (x0, y0, x1, y1) in the top-k order (score descending, ties by lowest flat index)."""
    maps = np.asarray(maps, np.float32)
    _, h, w = maps.shape
    heat = heat_map(maps[0]).reshape(-1)
    order = np.lexsort((np.arange(heat.size), -heat.astype(np.float64)))[:TOPK]
    disp = maps[1:5].transpose(1, 2, 0)
    start, end = disp[:, :, :2], disp[:, :, 2:]
    dist = np.sqrt(np.sum((start - end) ** 2, axis=-1))
    segs = []
    for idx in order:
        y, x = int(idx) // w, int(idx) % w
        if heat[idx] > np.float32(thr_v) and dist[y, x] > np.float32(thr_d):
            d = disp[y, x].astype(np.float64)
            segs.append([int(2.0 * (x + d[0])), int(2.0 * (y + d[1])), int(2.0 * (x + d[2])), int(2.0 * (y + d[3]))])
    return np.array(segs, np.int64).reshape(-1, 4)


def clip_line(W, H, x1, y1, x2, y2):
    """OpenCV's clipLine(Size(W, H), pt1, pt2) on int64 points -> (inside, x1, y1, x2, y2).  The second endpoint is
    moved with the first one's already clipped coordinates, so the result depends on the endpoint order."""
    right, bottom = W - 1, H - 1
    if W <= 0 or H <= 0:
        return False, x1, y1, x2, y2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += math.trunc(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += math.trunc(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += math.trunc(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += math.trunc(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def line_pixels(W, H, x1, y1, x2, y2):
    """[(x, y)] that cv2.line(img, (x1, y1), (x2, y2), color, 1, LINE_8) sets on an H x W image: clipLine when an
    endpoint is outside, then LineIterator(connectivity 8, leftToRight): endpoints swapped when x2 < x1, Bresenham
    along the major axis with err = D - 2d, a minor step whenever err < 0 before the update."""
    x1, y1, x2, y2 = int(x1), int(y1), int(x2), int(y2)
    if not (0 <= x1 < W and 0 <= x2 < W and 0 <= y1 < H and 0 <= y2 < H):
        ok, x1, y1, x2, y2 = clip_line(W, H, x1, y1, x2, y2)
        if not ok:
            return []
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, y2 - y1
    sy = -1 if dy < 0 else 1
    dy = abs(dy)
    vert = dy > dx
    big, small = (dy, dx) if vert else (dx, dy)
    err = big - 2 * small
    x, y, out = x1, y1, []
    for _ in range(big + 1):
        out.append((x, y))
        minor = err < 0
        err += -2 * small + (2 * big if minor else 0)
        if vert:
            y += sy
            x += 1 if minor else 0
        else:
            x += 1
            y += sy if minor else 0
    return out


def random_segments(n, H, W, seed=0):
    """Off-image, reversed, degenerate, horizontal, vertical and diagonal segments with endpoints up to 60 px out."""
    rs = np.random.RandomState(seed)
    p = np.stack([rs.randint(-60, W + 60, n), rs.randint(-60, H + 60, n),
                  rs.randint(-60, W + 60, n), rs.randint(-60, H + 60, n)], 1)
    k = np.arange(n) % 8
    p[k == 0, 2:] = p[k == 0, :2]                                      # a point
    p[k == 1, 3] = p[k == 1, 1]                                        # horizontal
    p[k == 2, 2] = p[k == 2, 0]                                        # vertical
    p[k == 3, 3] = p[k == 3, 1] + (p[k == 3, 2] - p[k == 3, 0])        # diagonal
    p[k == 4, 3] = p[k == 4, 1] - (p[k == 4, 2] - p[k == 4, 0])        # anti-diagonal
    r = p[k == 5]
    p[k == 5] = r[:, [2, 3, 0, 1]]                                     # reversed copies of the next rows
    return p.astype(np.int64)


def draw_lines(H, W, segs):
    """uint8 [H, W] map with 255 on the pixels of every segment (x0, y0, x1, y1), as apply_mlsd draws them."""
    out = np.zeros((H, W), np.uint8)
    for s in np.asarray(segs, np.int64).reshape(-1, 4):
        for x, y in line_pixels(W, H, *[int(v) for v in s]):
            out[y, x] = 255
    return out


def apply_mlsd(sd, img_u8, thr_v=0.1, thr_d=0.1, device="cpu"):
    """-> (uint8 [H, W] line map, segments, [5, H/2, W/2] map or None when the reference would raise)."""
    H, W = img_u8.shape[:2]
    if not size_supported(H, W):
        return np.zeros((H, W), np.uint8), np.zeros((0, 4), np.int64), None
    maps = network(sd, img_u8, device)
    segs = decode(maps, thr_v, thr_d)
    return draw_lines(H, W, segs), segs, maps


def near_ties(maps, thr_v=0.1, thr_d=0.1, tol=1e-6, end_tol=1e-6):
    """Decisions of `decode` on an fp32 map that a last-ulp difference in the sigmoid (or in the map) could flip ->
    dict of reasons -> list of flat map indices, plus 'segments': int64 [n, 4] every segment those cells can
    produce (both truncations of an endpoint within end_tol of an integer).  tol is absolute on the scores / distances.
    Checked: the 3x3 NMS (a neighbour within tol of the cell's heat), thr_v, the 200th / 201st score gap, thr_d and
    the endpoints."""
    maps = np.asarray(maps, np.float32)
    _, h, w = maps.shape
    heat = torch.sigmoid(torch.from_numpy(maps[0])).numpy().astype(np.float64)
    kept = heat_map(maps[0]).astype(np.float64)
    pad = np.pad(heat, 1, constant_values=-1.0)
    nbr = np.full((h, w), -1.0)
    for dy in range(3):
        for dx in range(3):
            if dy != 1 or dx != 1:
                nbr = np.maximum(nbr, pad[dy:dy + h, dx:dx + w])
    thr = float(np.float32(thr_v))
    live = heat > thr - tol                                       # cells whose NMS outcome can matter
    reasons = {"nms": np.flatnonzero((np.abs(heat - nbr) <= tol) & live),
               "thr_v": np.flatnonzero((np.abs(heat - thr) <= tol) & (kept > 0)),
               "topk": np.zeros(0, np.int64), "thr_d": np.zeros(0, np.int64), "endpoint": np.zeros(0, np.int64)}
    flat = kept.reshape(-1)
    cand = np.flatnonzero(flat > thr)
    if cand.size > TOPK:
        s = np.sort(flat[cand])[::-1]
        cut = s[TOPK - 1]
        if cut - s[TOPK] <= tol:
            reasons["topk"] = cand[np.abs(flat[cand] - cut) <= tol]
    disp = maps[1:5].transpose(1, 2, 0)
    dist = np.sqrt(np.sum((disp[:, :, :2] - disp[:, :, 2:]) ** 2, axis=-1)).astype(np.float64).reshape(-1)
    near_d = np.abs(dist[cand] - float(np.float32(thr_d))) <= tol
    reasons["thr_d"] = cand[near_d]
    ends = []
    for idx in cand:
        y, x = int(idx) // w, int(idx) % w
        d = disp[y, x].astype(np.float64)
        e = 2.0 * (np.array([x, y, x, y], np.float64) + d)
        if np.any(np.abs(e - np.round(e)) <= end_tol):
            ends.append(idx)
    reasons["endpoint"] = np.array(ends, np.int64)
    cells = sorted(set(np.concatenate([v for v in reasons.values()]).tolist()))
    segs = []
    for idx in cells:
        y, x = idx // w, idx % w
        d = disp[y, x].astype(np.float64)
        e = 2.0 * (np.array([x, y, x, y], np.float64) + d)
        lo, hi = np.trunc(e - end_tol), np.trunc(e + end_tol)
        for k in range(16):
            segs.append([int(hi[j] if (k >> j) & 1 else lo[j]) for j in range(4)])
    reasons["segments"] = np.array(segs, np.int64).reshape(-1, 4)
    return reasons


def exempt_mask(H, W, ties):
    """Pixels a near-tie decision can reach: every possibly drawn variant of a flagged segment, grown by one pixel."""
    m = draw_lines(H, W, ties["segments"]) > 0
    g = np.pad(m, 1)
    return np.max([g[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], axis=0)
