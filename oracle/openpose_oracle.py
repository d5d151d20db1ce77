"""CPU oracle for the OpenPose body annotator (pfd_b200/openpose.py): the fp32 body network, synthetic weights, numpy
restatements of the reference's resizes, decode (Body.__call__ after the network, openpose/body.py:43-229) and drawing
(util.draw_bodypose with cv2.ellipse2Poly / fillConvexPoly / circle), and a near-tie report for the decode's
comparisons.  Tests compare the GPU path with it and with cv2 / scipy themselves."""
from __future__ import annotations

import math
from typing import List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from pfd_b200 import openpose_tables as T

LIMBS = [[2, 3], [2, 6], [3, 4], [4, 5], [6, 7], [7, 8], [2, 9], [9, 10], [10, 11], [2, 12], [12, 13], [13, 14],
         [2, 1], [1, 15], [15, 17], [1, 16], [16, 18], [3, 17], [6, 18]]
PAF_CH = [[31, 32], [39, 40], [33, 34], [35, 36], [41, 42], [43, 44], [19, 20], [21, 22], [23, 24], [25, 26],
          [27, 28], [29, 30], [47, 48], [49, 50], [53, 54], [51, 52], [55, 56], [37, 38], [45, 46]]


# ----------------------------------------------------------------------------------------------------------------
# resizes (cv2.resize restated on the tables of openpose_tables)
# ----------------------------------------------------------------------------------------------------------------
def resize(x: np.ndarray, H: int, W: int, area: bool) -> np.ndarray:
    """cv2.resize(x, (W, H), INTER_AREA if area else INTER_LANCZOS4) of a 2-D uint8 or float32 map."""
    u8 = x.dtype == np.uint8
    h, w = x.shape
    plan = T.resize_plan(h, w, H, W, area, fixed=u8 and not area)
    if plan[0] == "copy":
        return x.copy()
    if plan[0] == "block":
        fy, fx = plan[1], plan[2]
        blk = x[:H * fy, :W * fx].reshape(H, fy, W, fx)
        if u8:
            s = blk.astype(np.int64).sum(axis=(1, 3))
            if fy == 2 and fx == 2:
                return ((s + 2) >> 2).astype(np.uint8)
            v = s.astype(np.float32) * np.float32(1.0 / (fy * fx))
            return np.clip(np.rint(v), 0, 255).astype(np.uint8)
        acc = np.zeros((H, W), np.float32)
        for a in range(fy):
            for b in range(fx):
                acc = (acc + blk[:, a, :, b]).astype(np.float32)
        return (acc * np.float32(1.0 / (fy * fx))).astype(np.float32)
    (iy, wy), (ix, wx) = plan[1], plan[2]
    if u8 and not area:                                   # LANCZOS4 on uint8: int16 weights, int32 sums, >> 22
        rows = (x.astype(np.int64)[:, ix] * wx[None]).sum(-1)            # [h, W]
        v = (rows[iy] * wy[:, :, None]).sum(1)                            # [H, W]
        v = (v + (1 << (2 * T.COEF_BITS - 1))) >> (2 * T.COEF_BITS)
        return np.clip(v, 0, 255).astype(np.uint8)
    xf = x.astype(np.float32)
    rows = np.zeros((h, W), np.float32)
    for j in range(ix.shape[1]):
        rows = (rows + xf[:, ix[:, j]] * wx[None, :, j]).astype(np.float32)
    out = np.zeros((H, W), np.float32)
    for k in range(iy.shape[1]):
        out = (out + wy[:, k, None] * rows[iy[:, k]]).astype(np.float32)
    if u8:
        return np.clip(np.rint(out), 0, 255).astype(np.uint8)
    return out


# ----------------------------------------------------------------------------------------------------------------
# network
# ----------------------------------------------------------------------------------------------------------------
def synth_state_dict(seed: int = 0, gain: float = 1.0):
    """Name-seeded synthetic bodypose_model weights: He-scaled convs, so activations stay O(1) through the 6 stages;
    the stage heads get `gain` so heatmaps have peaks above the 0.1 threshold."""
    from pfd_b200.openpose import BodyPose
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in BodyPose().state_dict().items():
        if k.endswith("weight"):
            fan_in = v.shape[1] * v.shape[2] * v.shape[3]
            t = torch.randn(v.shape, generator=g) * math.sqrt(2.0 / fan_in)
            if "Mconv7" in k or "conv5_5" in k:
                t = t * gain
            sd[k] = t
        else:
            sd[k] = 0.05 * torch.randn(v.shape, generator=g)
    return sd


def network(sd, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """bodypose_model.forward in fp32 on NCHW x (u8 / 256 - 0.5, BGR): (Mconv7_stage6_L1, Mconv7_stage6_L2), with the
    reference's ReLU rules (a ReLU after every conv except the stage heads; stage 6's heatmap head keeps it)."""
    from pfd_b200.openpose import VGG, _layers
    conv = lambda t, name: F.conv2d(t, sd[name + ".weight"], sd[name + ".bias"],      # noqa: E731
                                    padding=sd[name + ".weight"].shape[-1] // 2)
    h = x
    for v in VGG:
        h = F.max_pool2d(h, 2, 2) if v == "pool" else F.relu(conv(h, "model0." + v[0]))
    out1, cur = h, h
    for i in range(1, 7):
        res = []
        for L in (1, 2):
            t = cur
            layers = _layers(i, L)
            for j, (name, _, _, _) in enumerate(layers):
                t = conv(t, f"model{i}_{L}.{name}")
                if j < len(layers) - 1 or (i == 6 and L == 2):
                    t = F.relu(t)
            res.append(t)
        cur = torch.cat([res[0], res[1], out1], 1)
    return res[0], res[1]


def network_input(img_u8_rgb: np.ndarray) -> Tuple[np.ndarray, Tuple[int, int]]:
    """Body.__call__'s input (body.py:51-60) for one uint8 RGB HxWx3 image: (float32 NCHW BGR network input, (h, w))."""
    H, W, _ = img_u8_rgb.shape
    bgr = img_u8_rgb[:, :, ::-1]
    s = 0.5 * 368 / H
    h, w = int(H * s), int(W * s)
    area = (H * s + W * s) / (H + W) < 1
    small = np.stack([resize(np.ascontiguousarray(bgr[:, :, c]), h, w, area) for c in range(3)], 2)
    hp, wp = h + (-h) % 8, w + (-w) % 8
    pad = np.full((hp, wp, 3), 128, np.uint8)
    pad[:h, :w] = small
    return (np.transpose(pad.astype(np.float32), (2, 0, 1))[None] / 256 - 0.5).astype(np.float32), (h, w)


def maps_to_image(m: np.ndarray, h: int, w: int, H: int, W: int) -> np.ndarray:
    """One stage-6 channel [h8, w8] -> the full-size float32 map (x8 LANCZOS4, crop, smart_resize)."""
    up = resize(m.astype(np.float32), m.shape[0] * 8, m.shape[1] * 8, area=False)[:h, :w]
    return resize(np.ascontiguousarray(up), H, W, area=(H + W) / (h + w) < 1)


# ----------------------------------------------------------------------------------------------------------------
# decode and drawing (body.py:88-229, util.py:70-124)
# ----------------------------------------------------------------------------------------------------------------
def gaussian(m: np.ndarray) -> np.ndarray:
    import scipy.ndimage
    return scipy.ndimage.gaussian_filter(m, sigma=3)


def decode(heat: np.ndarray, paf: np.ndarray, H: int):
    """heat float64 [H,W,18], paf float64 [H,W,38] -> (candidate [N,4], subset [M,20]) as Body.__call__ computes them."""
    all_peaks, counter = [], 0
    for part in range(18):
        m = heat[:, :, part]
        b = gaussian(m)
        nb = [np.zeros_like(b) for _ in range(4)]
        nb[0][1:, :], nb[1][:-1, :], nb[2][:, 1:], nb[3][:, :-1] = b[:-1, :], b[1:, :], b[:, :-1], b[:, 1:]
        ys, xs = np.nonzero((b >= nb[0]) & (b >= nb[1]) & (b >= nb[2]) & (b >= nb[3]) & (b > 0.1))
        all_peaks.append([(int(x), int(y), float(m[y, x]), counter + i) for i, (x, y) in enumerate(zip(xs, ys))])
        counter += len(xs)
    conns = []
    for k, ((a, b), (cx, cy)) in enumerate(zip(LIMBS, PAF_CH)):
        A, Bc = all_peaks[a - 1], all_peaks[b - 1]
        if not A or not Bc:
            conns.append(None)
            continue
        cand = []
        for i, pa in enumerate(A):
            for j, pb in enumerate(Bc):
                vx, vy = pb[0] - pa[0], pb[1] - pa[1]
                norm = max(0.001, math.sqrt(vx * vx + vy * vy))
                ux, uy = vx / norm, vy / norm
                px = np.linspace(pa[0], pb[0], num=10)
                py = np.linspace(pa[1], pb[1], num=10)
                sx = np.array([paf[int(round(py[t])), int(round(px[t])), cx - 19] for t in range(10)])
                sy = np.array([paf[int(round(py[t])), int(round(px[t])), cy - 19] for t in range(10)])
                sm = sx * ux + sy * uy
                sc = sum(sm) / 10 + min(0.5 * H / norm - 1, 0)
                if np.count_nonzero(sm > 0.05) > 8 and sc > 0:
                    cand.append((i, j, sc))
        cand.sort(key=lambda c: c[2], reverse=True)
        used_i, used_j, conn = set(), set(), []
        for i, j, sc in cand:
            if i not in used_i and j not in used_j:
                conn.append((A[i][3], Bc[j][3], sc))
                used_i.add(i)
                used_j.add(j)
                if len(conn) >= min(len(A), len(Bc)):
                    break
        conns.append(conn)
    candidate = np.array([p for ps in all_peaks for p in ps], np.float64).reshape(-1, 4)
    subset = []
    for k, conn in enumerate(conns):
        if conn is None:
            continue
        ia, ib = LIMBS[k][0] - 1, LIMBS[k][1] - 1
        for idA, idB, sc in conn:
            hits = [r for r in range(len(subset)) if subset[r][ia] == idA or subset[r][ib] == idB][:2]
            if len(hits) == 1:
                row = subset[hits[0]]
                if row[ib] != idB:
                    row[ib] = idB
                    row[19] += 1
                    row[18] += candidate[int(idB), 2] + sc
            elif len(hits) == 2:
                r1, r2 = subset[hits[0]], subset[hits[1]]
                if not np.any((r1[:18] >= 0) & (r2[:18] >= 0)):
                    r1[:18] += r2[:18] + 1
                    r1[18:] += r2[18:]
                    r1[18] += sc
                    del subset[hits[1]]
                else:
                    r1[ib] = idB
                    r1[19] += 1
                    r1[18] += candidate[int(idB), 2] + sc
            elif k < 17:
                row = -np.ones(20)
                row[ia], row[ib], row[19] = idA, idB, 2
                row[18] = candidate[int(idA), 2] + candidate[int(idB), 2] + sc
                subset.append(row)
    subset = [r for r in subset if not (r[19] < 4 or r[18] / r[19] < 0.4)]
    return candidate, np.array(subset, np.float64).reshape(-1, 20)


def draw(candidate: np.ndarray, subset: np.ndarray, H: int, W: int) -> np.ndarray:
    """draw_poses(body only) with cv2 itself: uint8 [H,W,3] canvas."""
    import cv2
    canvas = np.zeros((H, W, 3), np.uint8)
    colors = T.color_table()
    for person in subset:
        kps = [None if c < 0 else (candidate[int(c), 0] / float(W), candidate[int(c), 1] / float(H))
               for c in person[:18]]
        for k, (a, b) in enumerate(LIMBS[:17]):
            p, q = kps[a - 1], kps[b - 1]
            if p is None or q is None:
                continue
            Y = np.array([p[0], q[0]]) * float(W)
            X = np.array([p[1], q[1]]) * float(H)
            mX, mY = np.mean(X), np.mean(Y)
            length = ((X[0] - X[1]) ** 2 + (Y[0] - Y[1]) ** 2) ** 0.5
            angle = math.degrees(math.atan2(X[0] - X[1], Y[0] - Y[1]))
            poly = cv2.ellipse2Poly((int(mY), int(mX)), (int(length / 2), 4), int(angle), 0, 360, 1)
            cv2.fillConvexPoly(canvas, poly, [int(c) for c in colors[k]])
        for i, kp in enumerate(kps):
            if kp is not None:
                cv2.circle(canvas, (int(kp[0] * W), int(kp[1] * H)), 4, [int(c) for c in colors[17 + i]], thickness=-1)
    return canvas


def planted_maps(people: List[np.ndarray], H: int, W: int, sigma: float = 4.0, width: float = 3.0, skip=()):
    """Heatmaps [H,W,18] (Gaussian bumps of height 0.9 at each keypoint; rows of NaN are absent parts) and PAFs
    [H,W,38] (unit vectors along each limb within `width` px of it) for known skeletons (people: [18, 2] x, y each).
    skip: per person, limb indices whose PAF is left out (a person missing its neck-nose link is assembled as two
    rows that the ear-shoulder links then merge)."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    heat = np.zeros((H, W, 18))
    paf = np.zeros((H, W, 38))
    for n, P in enumerate(people):
        for p in range(18):
            if not np.isnan(P[p, 0]):
                heat[:, :, p] = np.maximum(heat[:, :, p], 0.9 * np.exp(-((xx - P[p, 0]) ** 2 + (yy - P[p, 1]) ** 2)
                                                                       / (2 * sigma ** 2)))
        for k, ((a, b), (cx, cy)) in enumerate(zip(LIMBS, PAF_CH)):
            pa, pb = P[a - 1], P[b - 1]
            if np.isnan(pa[0]) or np.isnan(pb[0]) or (n < len(skip) and k in skip[n]):
                continue
            v = pb - pa
            ln = np.hypot(*v)
            if ln == 0:
                continue
            u = v / ln
            t = (xx - pa[0]) * u[0] + (yy - pa[1]) * u[1]
            d = np.abs((xx - pa[0]) * u[1] - (yy - pa[1]) * u[0])
            on = (t >= -width) & (t <= ln + width) & (d <= width)
            paf[on, cx - 19], paf[on, cy - 19] = u[0], u[1]
    return heat.astype(np.float32), paf.astype(np.float32)


def reference_maps(l1: np.ndarray, l2: np.ndarray, h: int, w: int, H: int, W: int):
    """Body.__call__'s map resizes with cv2 itself (body.py:72-86): stage-6 PAFs [38,h8,w8] and heatmaps [19,h8,w8] ->
    float64 heat [H,W,18] and paf [H,W,38]."""
    import cv2

    def one(m):
        up = cv2.resize(m, (m.shape[1] * 8, m.shape[0] * 8), interpolation=cv2.INTER_LANCZOS4)[:h, :w]
        area = (H + W) / (h + w) < 1
        return cv2.resize(np.ascontiguousarray(up), (W, H), interpolation=cv2.INTER_AREA if area else cv2.INTER_LANCZOS4)
    heat = np.stack([one(l2[c].astype(np.float32)) for c in range(18)], 2).astype(np.float64)
    paf = np.stack([one(l1[c].astype(np.float32)) for c in range(38)], 2).astype(np.float64)
    return heat, paf


def resized_size(H: int, W: int):
    s = 0.5 * 368 / H
    return int(H * s), int(W * s)


def near_ties(heat: np.ndarray, paf: np.ndarray, candidate: np.ndarray, subset: np.ndarray, H: int, W: int,
              rel: float = 1e-9):
    """Decisions of the decode and drawing that a last-bit difference in the maps or in atan2 could flip: blurred values
    within `rel` of 0.1 or of a 4-neighbour (the >= peak test), PAF sample products within `rel` of 0.05, limb
    angles within 1e-9 degree of an integer off the axes and diagonals (int()), and equal connection scores (the
    sort).  Returns a dict of counts; all zero means the reference's decisions are robust."""
    out = {"threshold": 0, "neighbour": 0, "paf": 0, "angle": 0, "score_tie": 0}
    for part in range(18):
        b = gaussian(heat[:, :, part])
        out["threshold"] += int((np.abs(b - 0.1) <= rel * 0.1).sum())
        nb = np.pad(b, 1)
        near = [np.abs(b - nb[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]) <= rel * np.abs(b)
                for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1))]
        out["neighbour"] += int(((near[0] | near[1] | near[2] | near[3]) & (b > 0.1)).sum())
    out["paf"] = int((np.abs(np.abs(paf) - 0.05) <= rel).sum())
    for person in subset:
        for a, bb in LIMBS[:17]:
            ia, ib = int(person[a - 1]), int(person[bb - 1])
            if ia < 0 or ib < 0:
                continue
            x1, y1 = candidate[ia, 0] / float(W) * float(W), candidate[ia, 1] / float(H) * float(H)
            x2, y2 = candidate[ib, 0] / float(W) * float(W), candidate[ib, 1] / float(H) * float(H)
            ex, ey = y1 - y2, x1 - x2
            if ex == 0 or ey == 0 or abs(ex) == abs(ey):
                continue
            ang = math.degrees(math.atan2(ex, ey))
            if abs(ang - round(ang)) <= 1e-9:
                out["angle"] += 1
    sc = subset[:, 18] if len(subset) else np.zeros(0)
    out["score_tie"] = int(len(sc) - len(np.unique(sc)))
    return out
