"""PiDiNet soft-edge annotator (the default method of ControlNet.preprocess type 'scribble') on the pfd_b200 kernels.

Mirrors lib/model_zoo/controlnet_annotator/pidinet: ``PiDiNet`` has the state-dict keys and shapes of ``pidinet()``
(model.py:663-666: config 'carv4', 60 channels, dil=24, sa=True) and stores the unconverted pixel-difference (PDC)
weights, as table5_pidinet.pth does, so the checkpoint loads with ``strict=True``.  ``apply`` computes ``apply_pidinet``
(pidinet/__init__.py:67-96) plus the ToTensor / repeat of controlnet.py:469-471 for a whole batch at once:

    pfd_hed_input_f16 (norm 0, scale 1)       ToPILImage quantisation, channel-last fp16 levels 0..255 (exact)
    im2col3x3 + pfd_gemm_f16                  init_block, a 'cd' 3x3 conv 3 -> 60; the BGR flip and the / 255 of
                                              apply_pidinet are folded into the packed weights (input channels
                                              permuted, weights divided by 255)
    pfd_pidinet_dw_f16                        each block's depthwise conv1 + ReLU (with the 2x2 max-pool of the first
                                              block of stages 2-4 fused in front)
    pfd_gemm_f16                              conv2 + x; in the pooling blocks one two-segment GEMM
                                              [relu(dw(p)) | p] @ [conv2 | shortcut]^T + shortcut bias
    pfd_pidinet_reduce_f16 / _cdcm_f16        CDCM: ReLU + 1x1 to 24, then the four dilated 3x3 convs on the tensor cores
    pfd_pidinet_side_f32                      CSAM + MapReduce -> the stage's pre-sigmoid side map
    pfd_pidinet_fuse_f32                      F.interpolate(bilinear), classifier, sigmoid, uint8 truncation, /255, RGB

The PDC weights are converted to plain depthwise kernels in fp32 when they are packed: 'cv' as is; 'cd' subtracts the sum
of the 9 taps from the centre (conv(x, w) - conv1x1(x, sum w)); 'ad' is w - w[3,0,1,6,4,2,7,8,5]; 'rd' becomes a 5x5
kernel (padding 2) with +w[1:] on the outer positions {0,2,4,10,14,20,22,24}, -w[1:] on the inner ones
{6,7,8,11,13,16,17,18} and 0 in the centre (w[0] is unused, as in the reference).  Layer i (0 = init_block) is
cd / ad / rd / cv for i % 4 = 0 / 1 / 2 / 3.

The network runs in fp16 with fp32 accumulation and no activation scale: its inputs are in [0, 1] and the block outputs
stay far inside the fp16 range.  Stage 1 runs with 64 channels instead of 60 (the GEMM needs multiples of 8); it has
no biases, so the four pad channels stay exactly 0.

Like the reference's module-global ``netNetwork``, the network is process-global and not part of any pipeline's state
dict: ``load_pidinet`` reads table5_pidinet.pth (it never downloads), ``set_network`` installs a module built elsewhere.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn

from . import native as nv
from .annotator import AnnotatorNetwork
from .modules import cached

# pidinet/__init__.py:7-11,68-71: pretrained/controlnet/preprocess/pidinet/table5_pidinet.pth relative to the working
# directory
DEFAULT_PATH = os.path.join("pretrained", "controlnet", "preprocess", "pidinet", "table5_pidinet.pth")
C0, DIL = 60, 24
STAGE_CH = (C0, 2 * C0, 4 * C0, 4 * C0)
PDC_ORDER = ("cd", "ad", "rd", "cv")
AD_PERM = [3, 0, 1, 6, 4, 2, 7, 8, 5]
RD_OUTER = [0, 2, 4, 10, 14, 20, 22, 24]
RD_INNER = [6, 7, 8, 11, 13, 16, 17, 18]
MIN_SIZE = 8                                       # three 2x2 floor pools must leave stage 4 non-empty


def _w(*shape):
    return nn.Parameter(torch.zeros(shape))


class _Conv(nn.Module):
    """A conv's parameters only (weight, optional bias)."""

    def __init__(self, cout, cin, k, bias):
        super().__init__()
        self.weight = _w(cout, cin, k, k)
        if bias:
            self.bias = _w(cout)


class PDCBlock(nn.Module):
    """PDCBlock (model.py:441-463): [pool + shortcut], depthwise PDC conv1, ReLU, 1x1 conv2, + x."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        self.stride = stride
        if stride > 1:
            self.shortcut = _Conv(cout, cin, 1, True)
        self.conv1 = _Conv(cin, 1, 3, False)
        self.conv2 = _Conv(cout, cin, 1, False)


class CDCM(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.conv1 = _Conv(DIL, cin, 1, True)
        for j in range(4):
            setattr(self, f"conv2_{j + 1}", _Conv(DIL, DIL, 3, False))


class CSAM(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = _Conv(4, DIL, 1, True)
        self.conv2 = _Conv(1, 4, 3, False)


class MapReduce(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = _Conv(1, DIL, 1, True)


def _blocks():
    """[(name, stage, layer, cin, cout, stride)] of the 15 PDC blocks after init_block (layer 0)."""
    out, layer = [], 1
    for s in range(4):
        for j in range(3 if s == 0 else 4):
            first = j == 0 and s > 0
            out.append((f"block{s + 1}_{j + 1}", s, layer, STAGE_CH[s - 1] if first else STAGE_CH[s], STAGE_CH[s],
                        2 if first else 1))
            layer += 1
    return out


def convert_pdc(op: str, w: torch.Tensor) -> torch.Tensor:
    """PDC weights [C, I, 3, 3] -> the plain conv kernel (3x3, or 5x5 with padding 2 for 'rd'), in w's dtype."""
    c, i = w.shape[:2]
    f = w.reshape(c, i, 9)
    if op == "cv":
        return w.clone()
    if op == "cd":
        out = f.clone()
        out[:, :, 4] -= f.sum(-1)
        return out.reshape(w.shape)
    if op == "ad":
        return (f - f[:, :, AD_PERM]).reshape(w.shape)
    if op == "rd":
        out = torch.zeros((c, i, 25), dtype=w.dtype, device=w.device)
        out[:, :, RD_OUTER] = f[:, :, 1:]
        out[:, :, RD_INNER] = -f[:, :, 1:]
        return out.reshape(c, i, 5, 5)
    raise ValueError(f"unknown PDC type {op!r}")


def _pad_to(t: torch.Tensor, shape) -> torch.Tensor:
    out = torch.zeros(shape, dtype=t.dtype, device=t.device)
    out[tuple(slice(0, s) for s in t.shape)] = t
    return out


def _p8(c):
    return -(-c // 8) * 8


def pack_cdcm(weights) -> torch.Tensor:
    """CDCM's four [24, 24, 3, 3] dilated-conv weights -> fp16 mma.m16n8k16 B fragments [54, 3, 32, 4]
    (pfd_pidinet_cdcm_f16): K = (dilation, ky, kx, input channel) flattened, step s covers K rows 16s..16s+15, and lane
    g*4+t of n-tile j holds output channel 8j+g at step rows 2t, 2t+1, 2t+8, 2t+9."""
    w = torch.stack([x.detach().float() for x in weights])            # [4, n, c, ky, kx]
    k = w.permute(0, 3, 4, 2, 1).reshape(54, 2, 4, 2, 3, 8)           # [s, hi, t, e, j, g], K row = hi*8 + 2t + e
    return k.permute(0, 4, 5, 2, 1, 3).reshape(54, 3, 32, 4).to(torch.float16).contiguous()


class PiDiNet(nn.Module):
    """pidinet() (model.py:495-666, 'carv4', 60 channels, dil=24, sa=True) as a parameter holder; ``apply`` runs it on
    the GPU."""

    def __init__(self):
        super().__init__()
        self.init_block = _Conv(C0, 3, 3, False)
        for name, _, _, cin, cout, stride in _blocks():
            setattr(self, name, PDCBlock(cin, cout, stride))
        self.conv_reduces = nn.ModuleList([MapReduce() for _ in range(4)])
        self.attentions = nn.ModuleList([CSAM() for _ in range(4)])
        self.dilations = nn.ModuleList([CDCM(STAGE_CH[i]) for i in range(4)])
        self.classifier = _Conv(1, 4, 1, True)

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("PiDiNet is a parameter holder: call apply() (CUDA kernels only)")

    def _packed(self):
        """fp32 converted depthwise kernels, fp16 GEMM weights, and the fp32 CDCM / CSAM / fuse parameters."""
        def build():
            if not self.classifier.weight.is_cuda:
                raise RuntimeError("PiDiNet.apply needs the network on a CUDA device (call .to('cuda'))")
            f32 = lambda t: t.detach().float()                                    # noqa: E731
            # BGR input -> RGB channels; the input arrives as exact integer levels 0..255, so 1/255 goes here
            wi = convert_pdc(PDC_ORDER[0], f32(self.init_block.weight))[:, [2, 1, 0]] / 255.0
            wi = wi.permute(0, 2, 3, 1).reshape(C0, 27)                           # k = tap * 3 + c (im2col order)
            init = _pad_to(wi, (_p8(C0), 32)).to(torch.float16).contiguous()
            blocks = []
            for name, _, layer, cin, cout, stride in _blocks():
                blk = getattr(self, name)
                cp, op_ = _p8(cin), _p8(cout)
                wd = convert_pdc(PDC_ORDER[layer % 4], f32(blk.conv1.weight))    # [cin, 1, ks, ks]
                wd = _pad_to(wd.reshape(cin, -1).t(), (wd.shape[-1] ** 2, cp)).contiguous()
                w2 = _pad_to(f32(blk.conv2.weight).reshape(cout, cin), (op_, cp))
                bias = None
                if stride > 1:
                    ws = _pad_to(f32(blk.shortcut.weight).reshape(cout, cin), (op_, cp))
                    w2 = torch.cat([w2, ws], 1)
                    bias = _pad_to(f32(blk.shortcut.bias), (op_,)).to(torch.float16).contiguous()
                blocks.append((wd, w2.to(torch.float16).contiguous(), bias, stride))
            stages = []
            for i in range(4):
                cdcm, att, mr = self.dilations[i], self.attentions[i], self.conv_reduces[i]
                c = STAGE_CH[i]
                w1 = _pad_to(f32(cdcm.conv1.weight).reshape(DIL, c).t(), (_p8(c), DIL)).contiguous()
                b1 = f32(cdcm.conv1.bias).contiguous()
                wpk = pack_cdcm([getattr(cdcm, f"conv2_{j + 1}").weight for j in range(4)])
                prm = torch.cat([f32(att.conv1.weight).reshape(-1), f32(att.conv1.bias).reshape(-1),
                                 f32(att.conv2.weight).reshape(-1), f32(mr.conv.weight).reshape(-1),
                                 f32(mr.conv.bias).reshape(-1)]).contiguous()
                stages.append((w1, b1, wpk, prm))
            cls = torch.cat([f32(self.classifier.weight).reshape(4), f32(self.classifier.bias).reshape(1)]).contiguous()
            zeros = torch.zeros(3, device=cls.device, dtype=torch.float32)
            return init, blocks, stages, cls, zeros
        return cached(self, "pidinet", list(self.parameters()), build)

    @torch.no_grad()
    def apply(self, x: torch.Tensor, return_sides: bool = False):
        """x: CUDA [B,3,H,W] image in [0,1], fp16 or fp32 (H, W >= 8) -> float32 [B,3,H,W] soft-edge levels / 255
        (three equal channels), asynchronous on the current stream.  return_sides=True also returns the four fp32
        pre-sigmoid side maps [B,h_k,w_k] (the MapReduce outputs before the upsampling)."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"PiDiNet.apply: expected a [B,3,H,W] image, got {tuple(x.shape)}")
        B, _, H, W = x.shape
        if H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError(f"PiDiNet needs H and W >= {MIN_SIZE} (three 2x2 floor pools), got {H}x{W}")
        init, blocks, stages, cls, zeros = self._packed()
        h = nv.hed_input(x, zeros, 1.0)                      # u8 levels, exact in fp16 (u8 / 255 would round)
        col = nv.im2col3x3(h, init.shape[1])
        h = nv.linear(col.reshape(B * H * W, init.shape[1]), init).reshape(B, H, W, init.shape[0])
        feats = []
        for wd, w2, bias, stride in blocks:
            if stride > 1:
                feats.append(h)
                d, p = nv.pidinet_dw(h, wd, pool=True)
                h = nv.conv1x1(d, w2, bias, x2=p)
            else:
                h = nv.conv1x1(nv.pidinet_dw(h, wd), w2, residual=h)
        feats.append(h)
        sides = [nv.pidinet_side(nv.pidinet_cdcm(nv.pidinet_reduce(f, w1, b1), wpk), prm)
                 for f, (w1, b1, wpk, prm) in zip(feats, stages)]
        out = nv.pidinet_fuse(sides, cls, H, W)
        return (out, sides) if return_sides else out


_network: Optional[PiDiNet] = None  # set through NETWORK.set (set_network)
NETWORK = AnnotatorNetwork(__name__, PiDiNet, DEFAULT_PATH, "PiDiNet annotator")
set_network, load_pidinet, get_network, available = NETWORK.set, NETWORK.load, NETWORK.get, NETWORK.available


def preprocess_pidinet(x: torch.Tensor) -> torch.Tensor:
    """apply_pidinet + ToTensor + repeat for a CUDA [B,3,H,W] image in [0,1] -> float32 [B,3,H,W] (levels / 255)."""
    return NETWORK.on(x).apply(x)                              # apply_pidinet: netNetwork.to(device) (:80)
