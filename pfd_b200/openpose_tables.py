"""OpenCV resize and drawing tables for the OpenPose annotator (openpose.py), built on the host in float64 / float32
exactly as OpenCV 4.x builds them, so the device kernels reproduce cv2.resize and cv2.ellipse2Poly.

Every resize here is separable: out[y, x] = sum_k wy[y, k] * (sum_j wx[x, j] * src[iy[y, k], ix[x, j]]), summed left
to right without fused multiply-adds, which is the operation order of OpenCV's generic (non-IPP) resize for
INTER_LANCZOS4 and INTER_AREA.  An axis table is (idx int32 [D, T], w [D, T]); unused taps have weight 0.
"""
from __future__ import annotations

import math

import numpy as np

COEF_BITS = 11                         # INTER_RESIZE_COEF_BITS: uint8 LANCZOS4 weights are int(round(w * 2048))


def lanczos4(x: np.float32) -> np.ndarray:
    """cv2's interpolateLanczos4(x): float32 [8] weights for taps sx-3 .. sx+4 (sum normalised in float32)."""
    s45 = 0.70710678118654752440084436210485
    cs = ((1, 0), (-s45, -s45), (0, 1), (s45, -s45), (-1, 0), (s45, s45), (0, -1), (-s45, s45))
    x3 = np.float32(x + np.float32(3))
    y0 = -float(x3) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    c = np.zeros(8, np.float32)
    tot = np.float32(0)
    for i in range(8):
        yi = np.float32(x3 - np.float32(i))
        if abs(yi) >= np.float32(1e-6):
            y = -float(yi) * math.pi * 0.25
            c[i] = np.float32((cs[i][0] * s0 + cs[i][1] * c0) / (y * y))
        else:
            c[i] = np.float32(1e30)
        tot = np.float32(tot + c[i])
    inv = np.float32(np.float32(1) / tot)
    return (c * inv).astype(np.float32)


def lanczos_axis(S: int, D: int, fixed: bool):
    """INTER_LANCZOS4 along one axis, S -> D: source position (dx + 0.5) * S/D - 0.5 in float, taps clamped to the
    edge (replicate).  fixed=True gives uint8 resize's int16 weights (saturate_cast<short>(w * 2048))."""
    scale = 1.0 / (D / S)
    idx = np.zeros((D, 8), np.int32)
    w = np.zeros((D, 8), np.int32 if fixed else np.float32)
    for d in range(D):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(math.floor(f))
        f = np.float32(f - np.float32(s))
        c = lanczos4(f)
        idx[d] = np.clip(np.arange(s - 3, s + 5), 0, S - 1)
        w[d] = np.rint(c.astype(np.float64) * (1 << COEF_BITS)).astype(np.int32) if fixed else c
    return idx, w


def area_axis(S: int, D: int):
    """INTER_AREA along one axis for S >= D (cv2's computeResizeAreaTab): float32 weights over the source cells each
    destination cell covers, in increasing source order."""
    scale = 1.0 / (D / S)
    rows = []
    for d in range(D):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, S - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, S - 1)
        s1 = min(s1, s2)
        taps = []
        if s1 - f1 > 1e-3:
            taps.append((s1 - 1, np.float32((s1 - f1) / cell)))
        for s in range(s1, s2):
            taps.append((s, np.float32(1.0 / cell)))
        if f2 - s2 > 1e-3:
            taps.append((s2, np.float32(min(min(f2 - s2, 1.0), cell) / cell)))
        rows.append(taps)
    T = max(len(r) for r in rows)
    idx = np.zeros((D, T), np.int32)
    w = np.zeros((D, T), np.float32)
    for d, taps in enumerate(rows):
        for t, (s, a) in enumerate(taps):
            idx[d, t], w[d, t] = s, a
        idx[d, len(taps):] = taps[-1][0]
    return idx, w


def resize_plan(h: int, w: int, H: int, W: int, area: bool, fixed: bool):
    """How cv2.resize maps an h x w image to H x W with INTER_AREA (area=True) or INTER_LANCZOS4.
    Returns ('copy',), ('block', fy, fx) for an integer-factor area reduction (resizeAreaFast), or
    ('sep', (iy, wy), (ix, wx)) with separable tables."""
    if (h, w) == (H, W):
        return ("copy",)
    if area:
        sy, sx = 1.0 / (H / h), 1.0 / (W / w)
        if sy < 1 or sx < 1:
            raise NotImplementedError(f"INTER_AREA enlargement {h}x{w} -> {H}x{W} is not used by the annotator")
        iy, ix = int(round(sy)), int(round(sx))
        if abs(sy - iy) < np.finfo(np.float64).eps and abs(sx - ix) < np.finfo(np.float64).eps:
            return ("block", iy, ix)
        return ("sep", area_axis(h, H), area_axis(w, W))
    return ("sep", lanczos_axis(h, H, fixed), lanczos_axis(w, W, fixed))


# cv2's SinTable (drawing.cpp): sin of 0..450 degrees, stored as 7-decimal float literals
SIN_TABLE = np.array([round(math.sin(math.radians(i)), 7) for i in range(451)], np.float32)

# draw_bodypose's colours (util.py:95-97): circles use them as they are, limbs int(c * 0.6)
COLORS = [[255, 0, 0], [255, 85, 0], [255, 170, 0], [255, 255, 0], [170, 255, 0], [85, 255, 0], [0, 255, 0],
          [0, 255, 85], [0, 255, 170], [0, 255, 255], [0, 170, 255], [0, 85, 255], [0, 0, 255], [85, 0, 255],
          [170, 0, 255], [255, 0, 255], [255, 0, 170], [255, 0, 85]]


def color_table() -> np.ndarray:
    """uint8 [35, 3]: 17 limb colours int(c * 0.6), then 18 keypoint colours."""
    limbs = [[int(float(c) * 0.6) for c in col] for col in COLORS[:17]]
    return np.array(limbs + COLORS, np.uint8)
