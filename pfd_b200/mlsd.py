"""M-LSD line annotator (ControlNet.preprocess types 'mlsd' and 'mlsd_v11p') on the pfd_b200 kernels.

Mirrors lib/model_zoo/controlnet_annotator/mlsd: ``MLSD`` has the state-dict keys and shapes of MobileV2_MLSD_Large
(models/mbv2_mlsd_large.py, 362 keys, 1,533,680 parameters), so mlsd_large_512_fp32.pth loads with ``strict=True``.
``apply`` computes apply_mlsd (mlsd/__init__.py:56-81) with pred_lines (utils.py:49-88) at the image's own size, plus
the ToTensor / repeat of controlnet.py:378-386, for a whole batch at once:

    pfd_mlsd_input_f16                      ToPILImage quantisation, concat(rgb, ones) as exact fp16 levels
                                            [u8 - 127.5, 1 - 127.5]; the 1 / 127.5 lives in the stem weights
    pfd_gemm_f16 (3x3, stride 2, tap_off 1) the stem ConvBNReLU6 with the TFLite pad (F.pad(x, (0,1,0,1)), padding 0)
    pfd_gemm_f16 (1x1) + pfd_mlsd_dw_f16    each inverted residual: expand (ReLU), depthwise 3x3 (ReLU6 on its input
                                            and output), project (+ x)
    pfd_gemm_f16 + pfd_mlsd_upsample_f16    BlockTypeA: both 1x1 convs write straight into their channel halves of
                                            the concat buffer (the upsampled one through a low-resolution temporary)
    pfd_gemm_f16 (3x3)                      BlockTypeB: relu(conv1(x)) + x in the GEMM epilogue (fp16 add after the
                                            rounding, the reference's order), then conv2
    pfd_gemm_f16 x 25                       BlockTypeC's dilation-5 conv: out[5i+p, 5j+q] only reads x[5i'+p, 5j'+q],
                                            so it is 25 plain 3x3 convs, one per phase (p, q), on strided views
    pfd_mlsd_head_f32                       block23.conv3's rows 7..11 in fp32 -> [B,5,H/2,W/2] fp32 maps
    pfd_mlsd_decode_f32                     sigmoid, 3x3 NMS, top-200, thr_v / thr_d, float64 endpoints (on the device)
    pfd_mlsd_draw_f32                       cv2.line(..., 1, LINE_8): OpenCV's clipLine + 8-connected LineIterator

BN (eval, eps 1e-5) is folded into the conv weights and biases in fp32 when the weights are packed.  The packing is
keyed on the parameters and buffers, so ``load_state_dict`` into the live module takes effect on the next call.

The reference swallows every exception inside pred_lines and returns a blank map.  Three cases raise there, and they
give exact zeros here too: image sizes the decoder cannot concatenate (floor(H/2) or floor(W/2) not a multiple of 8,
that is H or W mod 16 not in {0, 1}) and maps with fewer than 200 cells (torch.topk) are decided from the shape,
without running the network; an image with no surviving segment simply draws nothing.

Like the reference's module-global ``mlsdmodel``, the network is process-global and not part of any pipeline's state
dict: ``load_mlsd`` reads mlsd_large_512_fp32.pth (it never downloads), ``set_network`` installs a module built
elsewhere.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn

from . import native as nv
from .annotator import AnnotatorNetwork
from .modules import cached, fp16, pack_conv

# mlsd/__init__.py:11-16,59: pretrained/controlnet/preprocess/mlsd/mlsd_large_512_fp32.pth relative to the working
# directory
DEFAULT_PATH = os.path.join("pretrained", "controlnet", "preprocess", "mlsd", "mlsd_large_512_fp32.pth")
TOPK = nv.PFD_MLSD_TOPK
BN_EPS = 1e-5
TRUNK = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1))   # t, c, n, s
FPN = (1, 3, 6, 10, 13)
DECODER = (("block15", 64, 96, False), ("block17", 32, 64, True), ("block19", 24, 64, True),
           ("block21", 16, 64, True))                                                 # name, in_c1, in_c2, upscale
KEEP = slice(7, 12)                      # block23.conv3 rows the decode reads: centre, start x, y, end x, y
STEM_CIN = 16                            # rgb, ones and 12 zero channels (the GEMM's 3x3 path needs C >= 16)


def size_supported(H: int, W: int) -> bool:
    """True when the reference's pred_lines runs on an H x W image (see the module docstring)."""
    h, w = H // 2, W // 2
    return h > 0 and w > 0 and h % 8 == 0 and w % 8 == 0 and h * w >= TOPK


class _Conv(nn.Module):
    def __init__(self, cout, cin, k, bias):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(cout, cin, k, k))
        if bias:
            self.bias = nn.Parameter(torch.zeros(cout))


class _BN(nn.Module):
    """BatchNorm2d's parameters and buffers only."""

    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))


def _cbn(cout, cin, k, bias=False):
    return nn.Sequential(_Conv(cout, cin, k, bias), _BN(cout))


def trunk_layers():
    """[(feature index, inp, hidden, oup, stride, residual)] of the inverted residuals features[1..13]."""
    out, inp, i = [], 32, 1
    for t, c, n, s in TRUNK:
        for j in range(n):
            stride = s if j == 0 else 1
            out.append((i, inp, int(round(inp * t)), c, stride, stride == 1 and inp == c))
            inp, i = c, i + 1
    return out


class _InvertedResidual(nn.Module):
    def __init__(self, inp, hid, oup):
        super().__init__()
        layers = [_cbn(hid, inp, 1)] if hid != inp else []
        layers += [_cbn(hid, 1, 3), _Conv(oup, hid, 1, False), _BN(oup)]
        self.conv = nn.Sequential(*layers)


class _Backbone(nn.Module):
    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(_cbn(32, 4, 3), *[_InvertedResidual(inp, hid, oup)
                                                        for _, inp, hid, oup, _, _ in trunk_layers()])


class _BlockA(nn.Module):
    def __init__(self, in_c1, in_c2):
        super().__init__()
        self.conv1 = _cbn(64, in_c2, 1, True)
        self.conv2 = _cbn(64, in_c1, 1, True)


class _BlockB(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = _cbn(128, 128, 3, True)
        self.conv2 = _cbn(64, 128, 3, True)


class _BlockC(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = _cbn(64, 64, 3, True)
        self.conv2 = _cbn(64, 64, 3, True)
        self.conv3 = _Conv(16, 64, 1, True)


def fold_bn(conv: nn.Module, bn: nn.Module):
    """(weight, bias) of conv followed by eval-mode BN, in fp32."""
    f = lambda t: t.detach().float()                                              # noqa: E731
    scale = f(bn.weight) / torch.sqrt(f(bn.running_var) + BN_EPS)
    b = f(conv.bias) if getattr(conv, "bias", None) is not None else torch.zeros_like(scale)
    return f(conv.weight) * scale.reshape(-1, 1, 1, 1), (b - f(bn.running_mean)) * scale + f(bn.bias)


def _dilated5(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """relu(conv3x3(x, dilation 5, padding 5) + b) of x [B,h,w,C]: phase (p, q) of the output only reads phase (p, q)
    of the input, with a plain 3x3 / padding 1 conv, so each phase is one GEMM on strided views."""
    B, h, wd, _ = x.shape
    out = torch.empty((B, h, wd, w.shape[0]), device=x.device, dtype=torch.float16)
    for p in range(min(5, h)):
        for q in range(min(5, wd)):
            nv.conv3x3(x[:, p::5, q::5], w, b, act=nv.ACT_RELU, out=out[:, p::5, q::5])
    return out


class MLSD(nn.Module):
    """MobileV2_MLSD_Large (mbv2_mlsd_large.py:247-292) as a parameter holder; ``apply`` runs it on the GPU."""

    def __init__(self):
        super().__init__()
        self.backbone = _Backbone()
        for k, (name, c1, c2, _) in enumerate(DECODER):
            setattr(self, name, _BlockA(c1, c2))
            setattr(self, f"block{16 + 2 * k}", _BlockB())
        self.block23 = _BlockC()

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("MLSD is a parameter holder: call apply() (CUDA kernels only)")

    def _packed(self):
        """BN-folded fp16 GEMM weights with fp16 biases, fp32 depthwise weights [9, C] and biases, fp32 head."""
        def build():
            if not self.block23.conv3.weight.is_cuda:
                raise RuntimeError("MLSD.apply needs the network on a CUDA device (call .to('cuda'))")
            f = self.backbone.features
            w, b = fold_bn(f[0][0], f[0][1])
            stem = (pack_conv(w / 127.5, STEM_CIN), fp16(b))      # the input arrives as u8 - 127.5 (exact levels)
            trunk = []
            for i, inp, hid, oup, stride, res in trunk_layers():
                seq = f[i].conv
                expand = None
                if hid != inp:
                    w, b = fold_bn(seq[0][0], seq[0][1])
                    expand = (pack_conv(w), fp16(b))
                    seq = seq[1:]
                w, b = fold_bn(seq[0][0], seq[0][1])
                dw = (w.reshape(hid, 9).t().contiguous(), b.contiguous())
                w, b = fold_bn(seq[1], seq[2])
                trunk.append((i, stride, res, expand, dw, (pack_conv(w), fp16(b))))
            decoder = []
            for k, (name, _, _, up) in enumerate(DECODER):
                ba, bb = getattr(self, name), getattr(self, f"block{16 + 2 * k}")
                convs = [fold_bn(s[0], s[1]) for s in (ba.conv1, ba.conv2, bb.conv1, bb.conv2)]
                decoder.append((up, *[(pack_conv(w), fp16(b)) for w, b in convs]))
            c = self.block23
            dil, conv2 = [(pack_conv(w), fp16(b)) for w, b in (fold_bn(c.conv1[0], c.conv1[1]),
                                                            fold_bn(c.conv2[0], c.conv2[1]))]
            head = (c.conv3.weight.detach().float()[KEEP].reshape(5, -1).contiguous(),
                    c.conv3.bias.detach().float()[KEEP].contiguous())
            return stem, trunk, decoder, dil, conv2, head
        return cached(self, "mlsd", list(self.parameters()) + list(self.buffers()), build)

    @torch.no_grad()
    def network(self, x: torch.Tensor) -> torch.Tensor:
        """x: CUDA [B,3,H,W] image in [0,1] (fp16 / fp32) of a supported size -> fp32 [B,5,H/2,W/2]: the network's
        output channels 7..11 (centre logit, start x, y, end x, y displacements)."""
        stem, trunk, decoder, dil, conv2, head = self._packed()
        h = nv.conv3x3(nv.mlsd_input(x), *stem, stride=2, act=nv.ACT_RELU, tap_off=1)
        feats = []
        for i, stride, res, expand, dw, proj in trunk:
            t = nv.conv1x1(h, *expand, act=nv.ACT_RELU) if expand is not None else h
            t = nv.mlsd_dw(t, *dw, stride)
            h = nv.conv1x1(t, *proj, residual=h if res else None)
            if i in FPN:
                feats.append(h)
        x = feats[4]
        for (up, (w1, b1), (w2, b2), (wb1, bb1), (wb2, bb2)), a in zip(decoder, feats[3::-1]):
            B, hh, ww, _ = a.shape
            cat = torch.empty((B, hh, ww, 128), device=a.device, dtype=torch.float16)
            nv.conv1x1_into(a, w2, b2, cat[..., :64], act=nv.ACT_RELU)
            if up:
                nv.mlsd_upsample(nv.conv1x1(x, w1, b1, act=nv.ACT_RELU), cat[..., 64:])
            else:
                nv.conv1x1_into(x, w1, b1, cat[..., 64:], act=nv.ACT_RELU)
            t = nv.conv3x3(cat, wb1, bb1, act=nv.ACT_RELU, residual=cat)
            x = nv.conv3x3(t, wb2, bb2, act=nv.ACT_RELU)
        x = nv.conv3x3(_dilated5(x, *dil), *conv2, act=nv.ACT_RELU)
        return nv.mlsd_head(x, *head)

    @torch.no_grad()
    def apply(self, x: torch.Tensor, thr_v: float = 0.1, thr_d: float = 0.1, debug: bool = False):
        """x: CUDA [B,3,H,W] image in [0,1], fp16 or fp32 -> float32 [B,3,H,W] line map (1.0 on the lines, three equal
        channels), asynchronous on the current stream.  debug=True also returns a dict with the network's 'maps'
        (fp32 [B,5,H/2,W/2], None for unsupported sizes), 'segs' (int32 [B,200,4], x0, y0, x1, y1) and 'count' (int32
        [B]; rows of segs past count are unspecified), all on the device."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"MLSD.apply: expected a [B,3,H,W] image, got {tuple(x.shape)}")
        B, _, H, W = x.shape
        if not size_supported(H, W):
            out = torch.zeros((B, 3, H, W), device=x.device, dtype=torch.float32)
            info = {"maps": None, "segs": torch.zeros((B, TOPK, 4), device=x.device, dtype=torch.int32),
                    "count": torch.zeros((B,), device=x.device, dtype=torch.int32)}
            return (out, info) if debug else out
        maps = self.network(x)
        segs, count = nv.mlsd_decode(maps, thr_v, thr_d)
        out = nv.mlsd_draw(segs, count, H, W)
        return (out, {"maps": maps, "segs": segs, "count": count}) if debug else out


_network: Optional[MLSD] = None  # set through NETWORK.set (set_network)
NETWORK = AnnotatorNetwork(__name__, MLSD, DEFAULT_PATH, "M-LSD annotator")
set_network, load_mlsd, get_network, available = NETWORK.set, NETWORK.load, NETWORK.get, NETWORK.available


def preprocess_mlsd(x: torch.Tensor, thr_v: float = 0.1, thr_d: float = 0.1) -> torch.Tensor:
    """apply_mlsd + ToTensor + repeat for a CUDA [B,3,H,W] image in [0,1] -> float32 [B,3,H,W] (1.0 on the lines)."""
    if not available():
        raise NotImplementedError(
            "controlnet annotator 'mlsd' needs the M-LSD weights, which are not installed: put "
            f"mlsd_large_512_fp32.pth at {DEFAULT_PATH}, call pfd_b200.mlsd.load_mlsd(path) or "
            "pfd_b200.mlsd.set_network(net), or feed a ready control map (do_preprocess=False)")
    return NETWORK.on(x).apply(x, thr_v, thr_d)                # apply_mlsd: mlsdmodel.to(device) (:67)
