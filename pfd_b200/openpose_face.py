"""OpenPose face annotator (ControlNet.preprocess types 'openpose_withface' and 'openpose_withface_v11p') on the pfd_b200
kernels.

Mirrors OpenposeDetector.__call__(include_body=True, include_hand=False, include_face=True)
(controlnet_annotator/openpose/__init__.py:200-290): the body annotator of openpose.py, then per person util.faceDetect
(util.py:296-375), Face.__call__ and Face.compute_peaks_from_heatmaps (face.py:331-361) and draw_poses with
util.draw_facepose.  ``FacePose`` has the state-dict keys and shapes of FaceNet (face.py:11-277, 104 keys, 38,425,706
parameters).  For a whole batch at once:

    BodyPose.detect                 the body annotator up to its persons (openpose.py)
    pfd_openpose_face_boxes         util.faceDetect of every person in float64, compacted in (image, person) order
    (one host readback)             the face count and boxes: the count sizes the network's M and each crop's size
                                    picks its resize tables
    pfd_openpose_face_input_f16     per face: ToPILImage quantisation, BGR, the crop oriImg[y:y+w, x:x+w] (clipped at the
                                    image edge as numpy clips it), util.smart_resize to 384 x 384 on OpenCV's tables
                                    (uint8 LANCZOS4, INTER_AREA, INTER_AREA emulated by OpenCV's bilinear when the crop
                                    has a side below 384, or a copy), u8 / 256 - 0.5
    pfd_gemm_f16 (3x3) + pool       the VGG trunk to conv5_3_CPM (128 channels at 48 x 48) and stage 1's 1x1 convs
    pfd_im2col7x7_f16 + pfd_gemm_f16   stages 2-6 on the concat buffer [71 maps -> 72 | 128 features], all faces of the
                                    batch in one M, in chunks of FACE_CHUNK faces so the im2col workspace stays bounded
    pfd_openpose_head_f32           stage 6's last 1x1 conv in fp32
    pfd_openpose_face_peaks_f32     F.interpolate(bilinear, align_corners=True) to the crop size in fp32, per channel the
                                    first maximum above 0.05 in raster order
    pfd_openpose_face_draw_f32      per person its body, then its face dots (float32 normalisation, cv2.circle(r=3))

Unlike 'openpose', this type synchronises with the host once per call (the face count) and cannot be captured in a CUDA
graph.  Like the reference's annotator, the network is process-global: ``load_face`` reads facenet.pth (it never
downloads), ``set_network`` installs a module built elsewhere.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import native as nv
from . import openpose
from . import openpose_tables as T
from .annotator import AnnotatorNetwork
from .modules import cached, fp16, pack_conv
from .openpose import CIN, _Conv, _rows

# openpose/__init__.py:11,123-127: the face model next to the body model
DEFAULT_PATH = os.path.join("pretrained", "controlnet", "preprocess", "openpose", "facenet.pth")
SIZE, MAPS = 384, 71                       # Face.__call__'s w_size, FaceNet's heatmaps (background included)
MAPS_PAD, CAT = 72, 200                    # concat buffer [71 maps + 1 zero channel | 128 features]
FACE_CHUNK = 8                             # faces per network pass: 8 x 45 MB of 7x7 im2col rows

TRUNK = (("conv1_1", 3, 64), ("conv1_2", 64, 64), "pool", ("conv2_1", 64, 128), ("conv2_2", 128, 128), "pool",
         ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256), "pool",
         ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512),
         ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3_CPM", 512, 128))


def stage_layers(i: int):
    """(name, cin, cout, k) of stage i (1: conv6_1_CPM, conv6_2_CPM; 2-6: Mconv1-7), face.py:62-170."""
    if i == 1:
        return [("conv6_1_CPM", 128, 512, 1), ("conv6_2_CPM", 512, MAPS, 1)]
    return [(f"Mconv1_stage{i}", 199, 128, 7)] + [(f"Mconv{j}_stage{i}", 128, 128, 7) for j in (2, 3, 4, 5)] + \
        [(f"Mconv6_stage{i}", 128, 128, 1), (f"Mconv7_stage{i}", 128, MAPS, 1)]


def _cat_w(w: torch.Tensor) -> torch.Tensor:
    """A stage's first 7x7 weights [128, 199, 7, 7] with the input channels moved to the concat buffer's layout."""
    w = w.detach().float()
    out = w.new_zeros((w.shape[0], CAT, 7, 7))
    out[:, :MAPS], out[:, MAPS_PAD:] = w[:, :MAPS], w[:, MAPS:]
    return out


class FacePose(nn.Module):
    """FaceNet (openpose/face.py) as a parameter holder; ``network`` runs it on the GPU."""

    def __init__(self):
        super().__init__()
        for v in TRUNK:
            if v != "pool":
                setattr(self, v[0], _Conv(v[1], v[2], 3))
        for i in range(1, 7):
            for name, cin, cout, k in stage_layers(i):
                setattr(self, name, _Conv(cin, cout, k))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("FacePose is a parameter holder: call network() (CUDA kernels only)")

    def _packed(self):
        def build():
            if not self.conv1_1.weight.is_cuda:
                raise RuntimeError("FacePose.network needs the network on a CUDA device (call .to('cuda'))")
            trunk = [None if v == "pool" else
                     (pack_conv(getattr(self, v[0]).weight, CIN if v[1] < CIN else None), fp16(getattr(self, v[0]).bias))
                     for v in TRUNK]
            stages = []
            for i in range(1, 7):
                convs = [getattr(self, name) for name, _, _, _ in stage_layers(i)]
                first = convs[0].weight if i == 1 else _cat_w(convs[0].weight)
                mid = [(pack_conv(first), fp16(convs[0].bias))] + [(pack_conv(c.weight), fp16(c.bias)) for c in convs[1:-1]]
                last = convs[-1]
                if i < 6:
                    tail = _rows(last.weight, last.bias, MAPS_PAD)
                else:
                    tail = (last.weight.detach().float().reshape(MAPS, -1).contiguous(),
                            last.bias.detach().float().contiguous())
                stages.append((mid, tail))
            return trunk, stages
        return cached(self, "openpose_face", list(self.parameters()), build)

    @torch.no_grad()
    def network(self, inp: torch.Tensor) -> torch.Tensor:
        """inp: channel-last fp16 [F,384,384,16] face inputs -> fp32 [F,71,48,48]: Mconv7_stage6 (hs[-1], no ReLU).
        The faces run FACE_CHUNK at a time."""
        F = inp.shape[0]
        h, w = inp.shape[1] // 8, inp.shape[2] // 8
        maps = torch.empty((F, MAPS, h, w), device=inp.device, dtype=torch.float32)
        for f0 in range(0, F, FACE_CHUNK):
            self._chunk(inp[f0:f0 + FACE_CHUNK], maps[f0:f0 + FACE_CHUNK])
        return maps

    def _chunk(self, x: torch.Tensor, maps: torch.Tensor) -> None:
        trunk, stages = self._packed()
        for t in trunk[:-1]:
            x = nv.openpose_pool(x) if t is None else nv.conv3x3(x, *t, act=nv.ACT_RELU)
        B, h, w, _ = x.shape
        # every stage writes all 200 channels: the padded head row gives an exact zero in channel 71
        cat = torch.empty((B, h, w, CAT), device=x.device, dtype=torch.float16)
        feat = nv.conv3x3(x, *trunk[-1], act=nv.ACT_RELU, out=cat[..., MAPS_PAD:])
        for i, (mid, tail) in enumerate(stages, start=1):
            t = feat if i == 1 else cat
            for wgt, bias in mid:
                if wgt.shape[1] == t.shape[3]:
                    t = nv.conv1x1(t.contiguous(), wgt, bias, act=nv.ACT_RELU)
                else:
                    t = nv.linear(nv.im2col7x7(t), wgt, bias, act=nv.ACT_RELU).reshape(B, h, w, -1)
            if i < 6:
                nv.conv1x1_into(t, *tail, cat[..., :MAPS_PAD])
            else:
                nv.openpose_head(t, tail[0], tail[1], False, maps, 0)


_plans = {}


def _resize(ch: int, cw: int, device):
    """(plan, device tables) of util.smart_resize for a ch x cw crop: INTER_AREA when 768 / (ch + cw) < 1, else
    INTER_LANCZOS4, both on uint8."""
    key = (ch, cw, str(device))
    if key not in _plans:
        plan = T.resize_plan(ch, cw, SIZE, SIZE, area=2.0 * SIZE / (ch + cw) < 1, fixed=True)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)              # noqa: E731
        tabs = tuple((dev(i), dev(wt)) for i, wt in plan[1:]) if plan[0] in ("sep", "linear") else None
        _plans[key] = (plan, tabs)
    return _plans[key]


_colors = {}


def _color_table(device) -> torch.Tensor:
    """uint8 [106, 3]: the body's 35 colours (openpose_tables.color_table), then 71 x white for the face dots."""
    key = str(device)
    if key not in _colors:
        _colors[key] = torch.from_numpy(np.concatenate([T.color_table(), np.full((MAPS, 3), 255, np.uint8)])).to(device)
    return _colors[key]


_network: Optional[FacePose] = None  # set through NETWORK.set (set_network)
NETWORK = AnnotatorNetwork(__name__, FacePose, DEFAULT_PATH, "OpenPose face")
set_network, load_face, get_network, available = NETWORK.set, NETWORK.load, NETWORK.get, NETWORK.available


@torch.no_grad()
def apply(body: openpose.BodyPose, face: FacePose, x: torch.Tensor, debug: bool = False,
          body_maps: Optional[torch.Tensor] = None, face_maps=None):
    """The 'openpose_withface' annotator for a CUDA [B,3,H,W] image in [0,1] -> float32 [B,3,H,W] (colour / 255).
    body_maps: given body stage-6 maps (BodyPose.detect).  face_maps: a callable (face inputs fp16 [F,384,384,16],
    boxes int [F,6]) -> fp32 [F,71,48,48] that replaces FaceNet.  debug=True also returns the body's debug dict plus
    'face_boxes' (int32 [F,6] on the host: image, person, x, y, ch, cw), 'face_input', 'face_maps' (fp32
    [F,71,48,48]) and 'face_landmarks' (int32 [F,71,2], crop pixels, -1 where the channel has none)."""
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("preprocess type 'openpose_withface' reads the face count back to the host and cannot be "
                           "captured in a CUDA graph; type='openpose' can")
    B, _, H, W = x.shape
    info = body.detect(x, body_maps)
    P = body._plans(H, W, x.device)
    persons, npersons, xy = info["persons"], info["npersons"], info["peaks_xy"]
    boxes, count = nv.openpose_face_boxes(persons, npersons, xy, H, W)
    F = int(count.item())
    host = boxes[:F].cpu()
    if F == 0:
        out = nv.openpose_draw(persons, npersons, xy, H, W, P["sintab"], P["colors"])
        inp = maps = lmk = None
    else:
        inp = torch.empty((F, SIZE, SIZE, CIN), device=x.device, dtype=torch.float16)
        for f, (n, _, bx, by, ch, cw) in enumerate(host.tolist()):
            plan, tabs = _resize(ch, cw, x.device)
            nv.openpose_face_input(x, n, (bx, by, ch, cw), SIZE, plan, tabs, inp[f])
        maps = face.network(inp) if face_maps is None else face_maps(inp, host)
        lmk = nv.openpose_face_peaks(maps.contiguous(), boxes)
        out = nv.openpose_face_draw(persons, npersons, xy, H, W, P["sintab"], _color_table(x.device), boxes, lmk, F)
    if not debug:
        return out
    info.update(face_boxes=host, face_input=inp, face_maps=maps, face_landmarks=lmk)
    return out, info


def preprocess_openpose_face(x: torch.Tensor, debug: bool = False) -> torch.Tensor:
    """OpenposeModel.run_model(include_body=True, include_face=True) + ToTensor for a CUDA [B,3,H,W] image in [0,1]
    -> float32 [B,3,H,W].  The face count is read back to the host once per call, so this type cannot be captured in
    a CUDA graph (a capturing stream raises RuntimeError).  Zero faces give exactly the 'openpose' canvas."""
    if not available():
        raise NotImplementedError(
            "controlnet annotator 'openpose_withface' needs the OpenPose face weights, which are not installed: put "
            f"facenet.pth at {DEFAULT_PATH}, call pfd_b200.openpose_face.load_face(path) or "
            "pfd_b200.openpose_face.set_network(net); type='openpose' runs the body annotator alone")
    if not openpose.available():
        return openpose.preprocess_openpose(x)            # raises the body annotator's NotImplementedError
    return apply(openpose.NETWORK.on(x), NETWORK.on(x), x, debug=debug)
