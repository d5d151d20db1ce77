"""CPU oracle for the OpenPose face annotator (pfd_b200/openpose_face.py): the fp32 FaceNet, synthetic weights,
util.faceDetect, the crop and util.smart_resize (cv2 itself), Face.__call__'s bilinear map and
compute_peaks_from_heatmaps, Detector.detect_face's float32 normalisation and draw_poses with the face dots, plus a
near-tie report for the arg-max and > 0.05 decisions.  Tests compare the GPU path with it and with cv2 itself."""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import openpose_oracle as O


def synth_state_dict(seed: int = 0, gain: float = 1.0):
    """Name-seeded synthetic FaceNet weights: He-scaled convs, the stage heads (conv6_2_CPM, Mconv7) times `gain`."""
    from pfd_b200.openpose_face import FacePose
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in FacePose().state_dict().items():
        if k.endswith("weight"):
            t = torch.randn(v.shape, generator=g) * math.sqrt(2.0 / (v.shape[1] * v.shape[2] * v.shape[3]))
            sd[k] = t * gain if ("Mconv7" in k or "conv6_2" in k) else t
        else:
            sd[k] = 0.05 * torch.randn(v.shape, generator=g)
    return sd


def network(sd, x: torch.Tensor) -> torch.Tensor:
    """FaceNet.forward in fp32 on NCHW x (u8 / 256 - 0.5, BGR) -> hs[-1] [N,71,48,48]."""
    from pfd_b200.openpose_face import TRUNK, stage_layers
    conv = lambda t, name: F.conv2d(t, sd[name + ".weight"], sd[name + ".bias"],        # noqa: E731
                                    padding=sd[name + ".weight"].shape[-1] // 2)
    h = x
    for v in TRUNK:
        h = F.max_pool2d(h, 2, 2) if v == "pool" else F.relu(conv(h, v[0]))
    feat, cur = h, h
    for i in range(1, 7):
        layers = stage_layers(i)
        t = cur
        for j, (name, _, _, _) in enumerate(layers):
            t = conv(t, name)
            if j < len(layers) - 1:
                t = F.relu(t)
        cur = torch.cat([t, feat], 1)
    return t


def planted_face_maps(seed):
    """71 x 48 x 48 planted face maps: a Gaussian bump per channel (height 0.1-0.9), channel 5 everywhere <= 0.05 and
    channel 9's bump at map column 0 (its landmark is at crop column 0, which detect_face maps to -1)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:48, 0:48].astype(np.float64)
    m = np.zeros((71, 48, 48))
    for c in range(71):
        cx, cy = rng.uniform(2, 45, 2)
        if c == 9:
            cx = 0.0
        m[c] = rng.uniform(0.1, 0.9) * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * rng.uniform(1.0, 3.0) ** 2))
    m[5] = 0.04 * m[5] / m[5].max()
    return torch.from_numpy(m.astype(np.float32))


def face_box(kp: np.ndarray, H: int, W: int) -> Optional[Tuple[int, int, int]]:
    """util.faceDetect on one person's keypoints kp [18, 2] (image pixels, NaN rows absent) -> (x, y, w) or None."""
    ok = lambda p: not np.isnan(kp[p, 0])                                             # noqa: E731
    if not ok(0) or not any(ok(p) for p in (14, 15, 16, 17)):
        return None
    x0, y0 = float(kp[0, 0]), float(kp[0, 1])
    width = 0.0
    for p, k in ((14, 3.0), (15, 3.0), (16, 1.5), (17, 1.5)):
        if ok(p):
            d = max(abs(x0 - float(kp[p, 0])), abs(y0 - float(kp[p, 1])))
            width = max(width, d * k)
    x, y = max(x0 - width, 0.0), max(y0 - width, 0.0)
    w1 = w2 = width * 2
    if x + width > W:
        w1 = W - x
    if y + width > H:
        w2 = H - y
    width = min(w1, w2)
    return (int(x), int(y), int(width)) if width >= 20 else None


def person_keypoints(candidate: np.ndarray, row: np.ndarray) -> np.ndarray:
    kp = np.full((18, 2), np.nan)
    for p in range(18):
        if row[p] >= 0:
            kp[p] = candidate[int(row[p]), :2]
    return kp


def face_input(bgr: np.ndarray, box) -> Tuple[np.ndarray, np.ndarray]:
    """Face.__call__'s input for oriImg (uint8 BGR HxWx3) and box (x, y, w): (the crop, float32 [1,3,384,384])."""
    import cv2
    x, y, w = box
    crop = bgr[y:y + w, x:x + w]
    k = 768.0 / (crop.shape[0] + crop.shape[1])
    r = cv2.resize(crop, (384, 384), interpolation=cv2.INTER_AREA if k < 1 else cv2.INTER_LANCZOS4)
    return crop, (torch.from_numpy(r).permute(2, 0, 1)[None].float() / 256.0 - 0.5).numpy()


def heatmaps(hs: np.ndarray, ch: int, cw: int) -> np.ndarray:
    """F.interpolate(hs, (ch, cw), bilinear, align_corners=True) of hs [71,48,48] -> [71,ch,cw] (float32)."""
    return F.interpolate(torch.from_numpy(hs)[None].float(), (ch, cw), mode="bilinear", align_corners=True)[0].numpy()


def peaks(maps: np.ndarray) -> np.ndarray:
    """compute_peaks_from_heatmaps per channel: int [71, 2] (x, y) of the first maximum above 0.05, -1 where none."""
    out = np.full((maps.shape[0], 2), -1, np.int64)
    for c in range(maps.shape[0]):
        m = maps[c]
        if (m > 0.05).any():
            i = int(np.argmax(np.where(m > 0.05, m, -np.inf)))
            out[c] = (i % m.shape[1], i // m.shape[1])
    return out


def near_ties(maps: np.ndarray, rel: float = 4e-6) -> List[int]:
    """Channels whose decisions a last-bit difference in the bilinear map could flip: a second position within `rel`
    of the maximum, or the maximum within `rel` of the 0.05 threshold."""
    out = []
    for c in range(maps.shape[0]):
        m = maps[c]
        top = float(m.max())
        tol = rel * max(abs(top), 0.05)
        if abs(top - 0.05) <= tol or ((m >= top - tol).sum() > 1 and top > 0.05 - tol):
            out.append(c)
    return out


def landmarks_to_pixels(lmk: np.ndarray, box, H: int, W: int) -> List[Tuple[int, int]]:
    """detect_face's float32 normalisation, then draw_facepose's int(x * W): the dots that are drawn."""
    x, y, W, H = int(box[0]), int(box[1]), int(W), int(H)       # python ints keep numpy's arithmetic in float32
    p = lmk[lmk[:, 0] >= 0].astype(np.float32)
    px = np.where(p[:, 0] < 1e-6, -1, p[:, 0] + x) / float(W)
    py = np.where(p[:, 1] < 1e-6, -1, p[:, 1] + y) / float(H)
    dots = [(int(a * W), int(b * H)) for a, b in zip(px.astype(np.float32), py.astype(np.float32))]
    return [(a, b) for a, b in dots if a > 0.01 and b > 0.01]


def draw(candidate: np.ndarray, subset: np.ndarray, dots: List[List[Tuple[int, int]]], H: int, W: int) -> np.ndarray:
    """draw_poses(body and face) with cv2 itself: per person its body (openpose_oracle.draw, every colour of which is
    non-black), then its face dots as white filled circles of radius 3."""
    import cv2
    canvas = np.zeros((H, W, 3), np.uint8)
    for i in range(len(subset)):
        body = O.draw(candidate, subset[i:i + 1], H, W)
        on = body.any(2)
        canvas[on] = body[on]
        for x, y in dots[i]:
            cv2.circle(canvas, (x, y), 3, (255, 255, 255), thickness=-1)
    return canvas
