"""OpenPose body annotator (ControlNet.preprocess types 'openpose' and 'openpose_v11p') on the pfd_b200 kernels.

Mirrors lib/model_zoo/controlnet_annotator/openpose with the body network only (OpenposeDetector.__call__ with
include_body=True, include_hand=False, include_face=False): ``BodyPose`` has the state-dict keys and shapes of
bodypose_model (model.py, 184 keys, 52,311,446 parameters).  ``apply`` computes Body.__call__ (body.py:43-229) and
draw_poses / util.draw_bodypose (util.py:70-124) plus the ToTensor of controlnet.py:396-406, for a whole batch at once:

    pfd_openpose_input_f16          ToPILImage quantisation, BGR, cv2.resize by 184 / H (INTER_AREA below 1, else
                                    INTER_LANCZOS4, on OpenCV's tables: openpose_tables.py), pad 128 to a multiple of 8,
                                    u8 / 256 - 0.5 (exact in fp16, the pad is exactly 0)
    pfd_gemm_f16 (3x3) + pool       the VGG trunk and the CPM convs (model0)
    pfd_gemm_f16                    each stage: the L1 and L2 branches' first convs as one GEMM (N = 256; they read the
                                    same input), then each branch; stage k's last 1x1 convs write straight into their
                                    slices of the concat buffer [L1 38 -> 40 | L2 19 -> 24 | out1 128] (192 channels,
                                    zero pad channels and zero weight columns)
    pfd_im2col7x7_f16 + pfd_gemm_f16   the 7x7 convs of stages 2-6
    pfd_openpose_head_f32           the stage-6 heads in fp32 (ReLU on the heatmaps, none on the PAFs, as the
                                    reference's no_relu_layers has it)
    pfd_openpose_resize_f32         LANCZOS4 x8, the crop to the resized image, then the heatmaps to H x W
    pfd_openpose_peaks_f32          float64 Gaussian (sigma 3) and peaks, at most PFD_OPENPOSE_MAX_PEAKS per part
    pfd_openpose_assemble_f32       PAF scoring (pointwise through the final resize), greedy matching, assembly
    pfd_openpose_draw_f32           ellipse2Poly + fillConvexPoly per limb, filled circle per keypoint

Everything runs on the current stream without a host synchronisation, so the call can be captured in a CUDA graph.
Limits that the reference does not have: at most PFD_OPENPOSE_MAX_PEAKS (128) peaks per (image, part) are kept, the
first in raster order ('peaks_total' in the debug dict counts all of them); where the reference raises IndexError
(one connection matching three person rows) the first two rows are used.

Like the reference's annotator, the network is process-global and not part of any pipeline's state dict:
``load_openpose`` reads body_pose_model.pth (it never downloads), ``set_network`` installs a module built elsewhere.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import native as nv
from . import openpose_tables as T
from .annotator import AnnotatorNetwork, read_state_dict
from .modules import cached, fp16, pack_conv

# openpose/__init__.py:11,123-127: pretrained/controlnet/preprocess/openpose/body_pose_model.pth relative to the working
# directory.  Only the body file is needed here (the reference also loads the hand and face networks).
DEFAULT_PATH = os.path.join("pretrained", "controlnet", "preprocess", "openpose", "body_pose_model.pth")
MAX_PEAKS = nv.PFD_OPENPOSE_MAX_PEAKS
BOXSIZE, STRIDE = 368, 8
CIN = 16                                   # b, g, r and 13 zero channels (the GEMM's 3x3 path needs C >= 16)
L1_PAD, L2_PAD, CAT = 40, 24, 192          # concat buffer [L1 | L2 | out1]

VGG = (("conv1_1", 3, 64), ("conv1_2", 64, 64), "pool", ("conv2_1", 64, 128), ("conv2_2", 128, 128), "pool",
       ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256), "pool",
       ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3_CPM", 512, 256), ("conv4_4_CPM", 256, 128))


def _layers(i: int, L: int):
    """(name, cin, cout, k) of branch L (1: PAFs, 38 out; 2: heatmaps, 19 out) of stage i (model.py:53-94)."""
    nout = 38 if L == 1 else 19
    if i == 1:
        return [(f"conv5_{j}_CPM_L{L}", 128, 128, 3) for j in (1, 2, 3)] + \
               [(f"conv5_4_CPM_L{L}", 128, 512, 1), (f"conv5_5_CPM_L{L}", 512, nout, 1)]
    return [(f"Mconv1_stage{i}_L{L}", 185, 128, 7)] + [(f"Mconv{j}_stage{i}_L{L}", 128, 128, 7) for j in (2, 3, 4, 5)] + \
        [(f"Mconv6_stage{i}_L{L}", 128, 128, 1), (f"Mconv7_stage{i}_L{L}", 128, nout, 1)]


class _Conv(nn.Module):
    def __init__(self, cin, cout, k):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(cout, cin, k, k))
        self.bias = nn.Parameter(torch.zeros(cout))


class _Seq(nn.Module):
    """A make_layers Sequential's parameters (only the convs have any)."""

    def __init__(self, convs):
        super().__init__()
        for name, cin, cout, k in convs:
            setattr(self, name, _Conv(cin, cout, k))


def _cat_w(w: torch.Tensor) -> torch.Tensor:
    """A stage's first 7x7 weights [128, 185, 7, 7] with the input channels moved to the concat buffer's layout."""
    w = w.detach().float()
    out = w.new_zeros((w.shape[0], CAT, 7, 7))
    out[:, :38], out[:, L1_PAD:L1_PAD + 19], out[:, L1_PAD + L2_PAD:] = w[:, :38], w[:, 38:57], w[:, 57:]
    return out


def _rows(w: torch.Tensor, b: torch.Tensor, n: int):
    """1x1 weights [N, C, 1, 1] / bias zero-padded to n output rows, as GEMM operands."""
    wp = w.detach().float().new_zeros((n,) + tuple(w.shape[1:]))
    bp = b.detach().float().new_zeros((n,))
    wp[:w.shape[0]], bp[:b.shape[0]] = w.detach().float(), b.detach().float()
    return pack_conv(wp), fp16(bp)


class BodyPose(nn.Module):
    """bodypose_model (openpose/model.py) as a parameter holder; ``apply`` runs it on the GPU."""

    def __init__(self):
        super().__init__()
        self.model0 = _Seq([(name, cin, cout, 3) for name, cin, cout in (v for v in VGG if v != "pool")])
        for i in range(1, 7):
            for L in (1, 2):
                setattr(self, f"model{i}_{L}", _Seq(_layers(i, L)))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("BodyPose is a parameter holder: call apply() (CUDA kernels only)")

    def _conv(self, i: int, L: int, j: int) -> _Conv:
        return getattr(getattr(self, f"model{i}_{L}"), _layers(i, L)[j][0])

    def _packed(self):
        def build():
            if not self.model0.conv1_1.weight.is_cuda:
                raise RuntimeError("BodyPose.apply needs the network on a CUDA device (call .to('cuda'))")
            trunk = []
            for v in VGG:
                if v == "pool":
                    trunk.append(None)
                    continue
                c = getattr(self.model0, v[0])
                trunk.append((pack_conv(c.weight, CIN if v[1] < CIN else None), fp16(c.bias)))
            stages = []
            for i in range(1, 7):
                a, b = self._conv(i, 1, 0), self._conv(i, 2, 0)
                wa = a.weight if i == 1 else _cat_w(a.weight)
                wb = b.weight if i == 1 else _cat_w(b.weight)
                first = (torch.cat([pack_conv(wa), pack_conv(wb)]), torch.cat([fp16(a.bias), fp16(b.bias)]))
                branches = []
                for L, pad in ((1, L1_PAD), (2, L2_PAD)):
                    n = len(_layers(i, L))
                    mid = [(pack_conv(c.weight), fp16(c.bias)) for c in (self._conv(i, L, j) for j in range(1, n - 1))]
                    last = self._conv(i, L, n - 1)
                    if i < 6:
                        tail = _rows(last.weight, last.bias, pad)
                    else:
                        tail = (last.weight.detach().float().reshape(last.weight.shape[0], -1).contiguous(),
                                last.bias.detach().float().contiguous())
                    branches.append((mid, tail))
                stages.append((first, branches))
            return trunk, stages
        return cached(self, "openpose", list(self.parameters()), build)

    @torch.no_grad()
    def network(self, inp: torch.Tensor) -> torch.Tensor:
        """inp: the channel-last fp16 [B,hp,wp,16] network input -> fp32 [B,57,hp/8,wp/8]: Mconv7_stage6_L1 (38 PAF
        channels, no ReLU), then relu(Mconv7_stage6_L2) (19 heatmap channels)."""
        trunk, stages = self._packed()
        x = inp
        for t in trunk[:-1]:
            x = nv.openpose_pool(x) if t is None else nv.conv3x3(x, *t, act=nv.ACT_RELU)
        B, h, w, _ = x.shape
        # every stage writes all 192 channels: its padded 1x1 rows give exact zeros in the pad channels
        cat = torch.empty((B, h, w, CAT), device=x.device, dtype=torch.float16)
        x = nv.conv3x3(x, *trunk[-1], act=nv.ACT_RELU, out=cat[..., L1_PAD + L2_PAD:])
        maps = torch.empty((B, 57, h, w), device=x.device, dtype=torch.float32)
        for i, (first, branches) in enumerate(stages, start=1):
            if i == 1:
                y = nv.conv3x3(x, *first, act=nv.ACT_RELU)
            else:
                y = nv.linear(nv.im2col7x7(cat), *first, act=nv.ACT_RELU).reshape(B, h, w, 256)
            outs = []
            for L, (mid, tail) in enumerate(branches):
                t = y[..., 128 * L:128 * (L + 1)].contiguous()
                for wgt, bias in mid:
                    if wgt.shape[1] == t.shape[3]:
                        t = nv.conv1x1(t, wgt, bias, act=nv.ACT_RELU)
                    elif wgt.shape[1] == 9 * t.shape[3]:
                        t = nv.conv3x3(t, wgt, bias, act=nv.ACT_RELU)
                    else:
                        t = nv.linear(nv.im2col7x7(t), wgt, bias, act=nv.ACT_RELU).reshape(B, h, w, -1)
                outs.append(t)
            for L, ((mid, tail), t) in enumerate(zip(branches, outs)):
                if i < 6:
                    lo = 0 if L == 0 else L1_PAD
                    nv.conv1x1_into(t, *tail, cat[..., lo:lo + tail[0].shape[0]])
                else:
                    nv.openpose_head(t, tail[0], tail[1], L == 1, maps, 0 if L == 0 else 38)
        return maps

    def _plans(self, H: int, W: int, device):
        """Per image size: resize plans with their device tables, the Gaussian, the sine and colour tables."""
        store = self.__dict__.setdefault("_pfd_op_plans", {})
        key = (H, W, str(device))
        if key not in store:
            s = BOXSIZE * 0.5 / H
            h, w = int(H * s), int(W * s)
            if h < STRIDE or w < STRIDE:
                raise ValueError(f"openpose: a {H}x{W} image resizes to {h}x{w}, smaller than the network's stride")
            hp, wp = h + (-h) % STRIDE, w + (-w) % STRIDE
            dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)              # noqa: E731
            tabs = lambda p: None if p[0] != "sep" else tuple((dev(i), dev(wt)) for i, wt in p[1:])   # noqa: E731
            k_in = (H * s + W * s) / (H + W)
            p_in = T.resize_plan(H, W, h, w, area=k_in < 1, fixed=True)
            up_y, up_x = T.lanczos_axis(hp // STRIDE, hp, False), T.lanczos_axis(wp // STRIDE, wp, False)
            p_up = ("sep", (up_y[0][:h], up_y[1][:h]), (up_x[0][:w], up_x[1][:w]))
            p_out = T.resize_plan(h, w, H, W, area=(H + W) / (h + w) < 1, fixed=False)
            x = np.arange(-12, 13, dtype=np.float64)
            phi = np.exp(-0.5 / 9.0 * x ** 2)
            phi = phi / phi.sum()
            store[key] = dict(h=h, w=w, hp=hp, wp=wp, p_in=p_in, t_in=tabs(p_in), p_up=p_up, t_up=tabs(p_up),
                              p_out=p_out, t_out=tabs(p_out), gauss=dev(phi[12:].copy()),
                              sintab=dev(T.SIN_TABLE), colors=dev(T.color_table()))
        return store[key]

    @torch.no_grad()
    def detect(self, x: torch.Tensor, maps: Optional[torch.Tensor] = None):
        """Body.__call__ for a CUDA [B,3,H,W] image in [0,1] without the drawing: the dict that apply(debug=True)
        returns.  maps (fp32 [B,57,h',w'], PAFs then heatmaps) replaces the network's stage-6 output, so planted or
        reference maps can be decoded."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"BodyPose.apply: expected a [B,3,H,W] image, got {tuple(x.shape)}")
        _, _, H, W = x.shape
        P = self._plans(H, W, x.device)
        if maps is None:
            maps = self.network(nv.openpose_input(x, P["h"], P["w"], P["hp"], P["wp"], P["p_in"], P["t_in"]))
        up = nv.openpose_resize(maps, 0, 57, P["h"], P["w"], P["p_up"], P["t_up"])
        heat = nv.openpose_resize(up, 38, 18, H, W, P["p_out"], P["t_out"])
        xy, score, total = nv.openpose_peaks(heat, P["gauss"])
        persons, pscore, npersons = nv.openpose_assemble(up, H, W, P["p_out"], P["t_out"], total, xy, score)
        return {"maps": maps, "heatmaps": heat, "peaks_xy": xy, "peaks_score": score, "peaks_total": total,
                "persons": persons, "person_score": pscore, "npersons": npersons}

    @torch.no_grad()
    def apply(self, x: torch.Tensor, debug: bool = False, maps: Optional[torch.Tensor] = None):
        """x: CUDA [B,3,H,W] image in [0,1], fp16 or fp32 -> float32 [B,3,H,W] pose map (colour / 255), asynchronous on
        the current stream.  debug=True also returns a dict of device tensors: 'maps' (fp32 [B,57,h',w'] stage-6 output,
        PAFs then heatmaps), 'heatmaps' (fp32 [B,18,H,W]), 'peaks_xy' (int32 [B,18,MAX_PEAKS,2]), 'peaks_score'
        (float64), 'peaks_total' (int32 [B,18], all peaks found), 'persons' (int32 [B,MAX_PERSONS,18], the peak index
        within each part or -1), 'person_score' (float64 [B,MAX_PERSONS,2]: total score, parts) and 'npersons'.
        maps: given stage-6 maps instead of the network's (see detect)."""
        info = self.detect(x, maps)
        P = self._plans(x.shape[2], x.shape[3], x.device)
        out = nv.openpose_draw(info["persons"], info["npersons"], info["peaks_xy"], x.shape[2], x.shape[3], P["sintab"],
                               P["colors"])
        return (out, info) if debug else out


def _read_state_dict(path: str):
    """read_state_dict, then the raw CMU keys ('conv1_1.weight', which the reference's util.transfer maps) get their
    block prefix back."""
    sd = read_state_dict(path)
    if not any(k.startswith("model0.") for k in sd):
        block = {name: blk for blk, seq in BodyPose().named_children() for name, _ in seq.named_children()}
        sd = {f"{block[k.rsplit('.', 1)[0]]}.{k}" if k.rsplit(".", 1)[0] in block else k: v for k, v in sd.items()}
    return sd


_network: Optional[BodyPose] = None  # set through NETWORK.set (set_network)
NETWORK = AnnotatorNetwork(__name__, BodyPose, DEFAULT_PATH, "OpenPose body", read=_read_state_dict)
set_network, load_openpose, get_network, available = NETWORK.set, NETWORK.load, NETWORK.get, NETWORK.available


def preprocess_openpose(x: torch.Tensor) -> torch.Tensor:
    """OpenposeModel.run_model(include_body=True) + ToTensor for a CUDA [B,3,H,W] image in [0,1] -> float32 [B,3,H,W]."""
    if not available():
        raise NotImplementedError(
            "controlnet annotator 'openpose' needs the OpenPose body weights, which are not installed: put "
            f"body_pose_model.pth at {DEFAULT_PATH}, call pfd_b200.openpose.load_openpose(path) or "
            "pfd_b200.openpose.set_network(net), or feed a ready control map (do_preprocess=False)")
    return NETWORK.on(x).apply(x)
