"""HED soft-edge annotator (ControlNet.preprocess types 'hed' / 'softedge_v11p') on the pfd_b200 kernels.

Mirrors lib/model_zoo/controlnet_annotator/hed/__init__.py: ``ControlNetHED`` has the state-dict keys and shapes of
``ControlNetHED_Apache2`` (:23-59), so the reference's ControlNetHED.pth loads with ``strict=True``, and ``apply``
computes ``apply_hed`` (:102-128) plus the ToTensor / repeat of controlnet.py:370-376 for a whole batch at once:

    pfd_hed_input_f16                        ToPILImage quantisation and `x - norm` (:52), channel-last fp16
    im2col3x3 + pfd_gemm_f16 (ReLU)          block1.convs.0 (3 input channels)
    pfd_gemm_f16 implicit-GEMM conv (ReLU)   the other 12 3x3 convolutions
    pfd_hed_pool_side_f16                    each block's 1x1 projection and the 2x2 max-pool into the next block
    pfd_hed_fuse_f32                         cv2.resize INTER_LINEAR, mean, sigmoid, uint8 truncation, /255, RGB

The reference runs the network in fp32 on 0..255 inputs; here it runs in fp16 with fp32 accumulation at activation
scale ``SCALE`` = 1/255: the input and every conv / projection bias are multiplied by SCALE when the weights are packed,
so every activation and side map is SCALE times the reference's (ReLU convolutions and max-pool are positively
homogeneous) and stays far from the fp16 range limit; the fuse kernel multiplies by 1/SCALE.

Like the reference's module-global ``netNetwork``, the network is process-global and not part of any pipeline's state
dict: ``load_hed`` reads ControlNetHED.pth (it never downloads), ``set_network`` installs a module built elsewhere.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn

from . import native as nv
from .annotator import AnnotatorNetwork
from .modules import Conv2d, IndexedSequential, cached, pack_conv, pad_cols

SCALE = 1.0 / 255.0
# hed/__init__.py:16,64,105: pretrained/controlnet/preprocess/hed/ControlNetHED.pth relative to the working directory
DEFAULT_PATH = os.path.join("pretrained", "controlnet", "preprocess", "hed", "ControlNetHED.pth")
_BLOCKS = [(3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3)]


class HEDBlock(nn.Module):
    """DoubleConvBlock (hed/__init__.py:23-39): `layers` 3x3 convs + ReLU, then a 1x1 projection to one channel."""

    def __init__(self, cin: int, cout: int, layers: int):
        super().__init__()
        self.convs = IndexedSequential(*[Conv2d(cin if i == 0 else cout, cout, 3, padding=1) for i in range(layers)])
        self.projection = Conv2d(cout, 1, 1)


class ControlNetHED(nn.Module):
    """ControlNetHED_Apache2 (hed/__init__.py:42-59) as a parameter holder; ``apply`` runs it on the GPU."""

    def __init__(self):
        super().__init__()
        self.norm = nn.Parameter(torch.zeros((1, 3, 1, 1)))
        for i, (cin, cout, layers) in enumerate(_BLOCKS):
            setattr(self, f"block{i + 1}", HEDBlock(cin, cout, layers))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("ControlNetHED is a parameter holder: call apply() (CUDA kernels only)")

    def blocks(self):
        return [getattr(self, f"block{i + 1}") for i in range(len(_BLOCKS))]

    def _packed(self):
        """fp16 conv weights in the GEMM's K order with biases times SCALE; fp32 projections (bias times SCALE)."""
        def build():
            if not self.norm.is_cuda:
                raise RuntimeError("ControlNetHED.apply needs the network on a CUDA device (call .to('cuda'))")
            convs, projs = [], []
            for bi, blk in enumerate(self.blocks()):
                layer = []
                for ci, conv in enumerate(blk.convs):
                    w = pack_conv(conv.weight)
                    if bi == 0 and ci == 0:
                        w = pad_cols(w)                                   # K = 27 -> 32 for the im2col GEMM
                    b = (conv.bias.detach().float() * SCALE).to(torch.float16).contiguous()
                    layer.append((w, b))
                convs.append(layer)
                pw = blk.projection.weight.detach().float().reshape(-1).contiguous()
                pb = (blk.projection.bias.detach().float() * SCALE).reshape(1).contiguous()
                projs.append((pw, pb))
            norm = self.norm.detach().float().reshape(3).contiguous()
            return convs, projs, norm
        return cached(self, "hed", list(self.parameters()), build)

    @torch.no_grad()
    def apply(self, x: torch.Tensor, return_sides: bool = False):
        """x: CUDA [B,3,H,W] image in [0,1], fp16 or fp32 -> float32 [B,3,H,W] soft-edge map (three equal channels),
        asynchronous on the current stream.  return_sides=True also returns the five fp32 side maps [B,h_k,w_k]
        (SCALE times the reference's projections)."""
        convs, projs, norm = self._packed()
        B, _, H, W = x.shape
        h = nv.hed_input(x, norm, SCALE)
        sides = []
        for bi, (layer, (pw, pb)) in enumerate(zip(convs, projs)):
            for ci, (w, b) in enumerate(layer):
                if bi == 0 and ci == 0:
                    kpad = w.shape[1]
                    Bh, Hh, Wh, _ = h.shape
                    col = nv.im2col3x3(h, kpad)
                    h = nv.linear(col.reshape(Bh * Hh * Wh, kpad), w, b, act=nv.ACT_RELU).reshape(Bh, Hh, Wh, w.shape[0])
                else:
                    h = nv.conv3x3(h, w, b, act=nv.ACT_RELU)
            side, pooled = nv.hed_pool_side(h, pw, pb, pool=bi < len(convs) - 1)
            sides.append(side)
            h = pooled
        out = nv.hed_fuse(sides, H, W, inv_scale=1.0 / SCALE)
        return (out, sides) if return_sides else out


_network: Optional[ControlNetHED] = None  # set through NETWORK.set (set_network)
NETWORK = AnnotatorNetwork(__name__, ControlNetHED, DEFAULT_PATH, "HED annotator")
set_network, load_hed, get_network = NETWORK.set, NETWORK.load, NETWORK.get


def preprocess_hed(x: torch.Tensor) -> torch.Tensor:
    """ControlNet.preprocess(x, type='hed') for a CUDA [B,3,H,W] image in [0,1] -> float32 [B,3,H,W]."""
    return NETWORK.on(x).apply(x)                              # apply_hed: netNetwork.to(device) (:111)
