"""AutoencoderKL on the pfd_b200 kernels — mirrors lib/model_zoo/autokl.py:14-54 and
lib/model_zoo/autokl_modules.py:59-202, 368-568.

`decode` is on the hot path (SURVEY.md §8 a17); `encode` (SURVEY.md §8 f4: img2img / image variation)
runs the Encoder on the same kernels — its stride-2 downsampling convs use the reference's asymmetric
F.pad(x, (0,1,0,1)) through the conv GEMM's `tap_off` (autokl_modules.py:69-76).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import native as nv
from .modules import Container, Conv2d, GroupNorm, pk_conv3, pk_conv3_small, pk_lin, pk_mat, pk_norm


def Normalize(c):
    return GroupNorm(32, c, eps=1e-6, affine=True)                       # autokl_modules.py:38-39


class ResnetBlock(nn.Module):
    """autokl_modules.py:82-141 (temb_channels=0, nin_shortcut when channels change)."""

    def __init__(self, in_channels, out_channels=None):
        super().__init__()
        out_channels = out_channels or in_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = Normalize(in_channels)
        self.conv1 = Conv2d(in_channels, out_channels, 3, padding=1)
        self.norm2 = Normalize(out_channels)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = Conv2d(out_channels, out_channels, 3, padding=1)
        if in_channels != out_channels:
            self.nin_shortcut = Conv2d(in_channels, out_channels, 1)


class AttnBlock(nn.Module):
    """autokl_modules.py:150-202."""

    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = Normalize(c)
        self.q, self.k, self.v, self.proj_out = Conv2d(c, c, 1), Conv2d(c, c, 1), Conv2d(c, c, 1), Conv2d(c, c, 1)


class _Resample(nn.Module):
    def __init__(self, c, stride):
        super().__init__()
        self.with_conv = True
        self.conv = Conv2d(c, c, 3, stride=stride, padding=1 if stride == 1 else 0)


class Encoder(nn.Module):
    """autokl_modules.py:368-459."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, **_):
        super().__init__()
        if attn_resolutions:
            raise NotImplementedError("pfd_b200 VAE encoder: attn_resolutions must be empty (autokl.yaml)")
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.conv_in = Conv2d(in_channels, ch, 3, padding=1)
        in_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        bi = ch
        for lvl in range(len(ch_mult)):
            lv = Container()
            lv.block = nn.ModuleList()
            lv.attn = nn.ModuleList()
            bi, bo = ch * in_mult[lvl], ch * ch_mult[lvl]
            for _ in range(num_res_blocks):
                lv.block.append(ResnetBlock(bi, bo))
                bi = bo
            if lvl != len(ch_mult) - 1:
                lv.downsample = _Resample(bi, 2)
            self.down.append(lv)
        self.mid = Container()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = ResnetBlock(bi), AttnBlock(bi), ResnetBlock(bi)
        self.norm_out = Normalize(bi)
        self.conv_out = Conv2d(bi, 2 * z_channels if double_z else z_channels, 3, padding=1)


class Decoder(nn.Module):
    """autokl_modules.py:462-568."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, **_):
        super().__init__()
        if attn_resolutions:
            raise NotImplementedError("pfd_b200 VAE decoder: attn_resolutions must be empty (autokl.yaml)")
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.out_ch = out_ch
        block_in = ch * ch_mult[-1]
        self.conv_in = Conv2d(z_channels, block_in, 3, padding=1)
        self.mid = Container()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = ResnetBlock(block_in), AttnBlock(block_in), ResnetBlock(block_in)
        self.up = nn.ModuleList()
        for lvl in reversed(range(self.num_resolutions)):
            up = Container()
            up.block = nn.ModuleList()
            up.attn = nn.ModuleList()
            block_out = ch * ch_mult[lvl]
            for _ in range(num_res_blocks + 1):
                up.block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
            if lvl != 0:
                up.upsample = _Resample(block_in, 1)
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = Conv2d(block_in, out_ch, 3, padding=1)


# ------------------------------------------------------------------------------------------------
def run_vae_resnet(rb: ResnetBlock, x: torch.Tensor) -> torch.Tensor:
    g, b = pk_norm(rb.norm1)
    h = nv.groupnorm(x, g, b, rb.norm1.eps, silu=True)
    w, bb = pk_conv3(rb.conv1)
    h = nv.conv3x3(h, w, bb)
    g, b = pk_norm(rb.norm2)
    h = nv.groupnorm(h, g, b, rb.norm2.eps, silu=True)
    if rb.in_channels != rb.out_channels:
        w, bb = pk_conv3(rb.conv2, rb.nin_shortcut)
        return nv.conv3x3(h, w, bb, skip=[x])
    w, bb = pk_conv3(rb.conv2)
    return nv.conv3x3(h, w, bb, residual=x)


def run_vae_attn(at: AttnBlock, x: torch.Tensor) -> torch.Tensor:
    """Single-head attention over H*W tokens with d = C (autokl_modules.py:178-202): scores are
    materialised in fp16 exactly like the reference's bmm -> *c^-0.5 -> softmax -> bmm."""
    B, H, W, C = x.shape
    N = H * W
    g, b = pk_norm(at.norm)
    hn = nv.groupnorm(x, g, b, at.norm.eps, silu=False).reshape(B * N, C)
    wq, bq = pk_lin(at.q)
    wk, bk = pk_lin(at.k)
    wv, bv = pk_lin(at.v)
    q = nv.linear(hn, wq, bq).reshape(B, N, C)
    k = nv.linear(hn, wk, bk).reshape(B, N, C)
    vt = torch.empty((B, C, N), device=x.device, dtype=torch.float16)
    nv.gemm_raw([(hn, 1, C, (C, C * N, C * N))], in_w=N, in_h=1, stride=1, W=N, H=1, NB=B, w=wv, N=C, K=C,
                bias=bv, out=vt, so=(C * N, 0, 0, 1, 0, N))
    # query rows are processed in chunks so the materialised fp16 scores stay <= ~512 MB (N = 36864 at 1536x1536
    # would otherwise need 2.7 GB per image inside every cached graph's memory pool)
    tq = max(128, min(N, ((1 << 28) // (B * N)) // 128 * 128))
    o = torch.empty((B, N, C), device=x.device, dtype=torch.float16)
    for r0 in range(0, N, tq):
        rows = min(tq, N - r0)
        sc = torch.empty((B, rows, N), device=x.device, dtype=torch.float16)
        nv.bmm_nt(q[:, r0:r0 + rows], k, out=sc, so=(rows * N, 0, 0, N, 0, 1))
        nv.softmax_(sc, float(C) ** -0.5)
        nv.bmm_nt(sc, vt, out=o[:, r0:r0 + rows], so=(N * C, 0, 0, C, 0, 1))
    w, bb = pk_lin(at.proj_out)
    return nv.linear(o.reshape(B * N, C), w, bb, residual=x.reshape(B * N, C)).reshape(B, H, W, C)


class AutoencoderKL(nn.Module):
    """autokl.py:14-54."""

    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, **_):
        super().__init__()
        assert ddconfig["double_z"]
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.quant_conv = Conv2d(2 * ddconfig["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.embed_dim = embed_dim

    @torch.no_grad()
    def encode(self, x: torch.Tensor, out_posterior: bool = False, post_scale: float = 1.0):
        """autokl.py:30-42: x NCHW in [0,1] -> x*2-1 -> Encoder (autokl_modules.py:436-459) -> quant_conv ->
        DiagonalGaussianDistribution -> posterior (out_posterior=True) or a sample [B, zc, H/8, W/8] (fp16;
        `post_scale` carries the pipeline's latent scale, pfd.py:266-273).  The sample's noise is drawn like
        the reference's: torch.randn(shape) on the CPU generator, then moved to the device."""
        enc = self.encoder
        if x.dtype not in (torch.float16, torch.float32):
            x = x.to(torch.float16)
        B = x.shape[0]
        nv.gn_reset()
        h = nv.nchw_to_nhwc(x, mul=2.0, add=-1.0)                          # [B,H,W,3]
        w, b = pk_conv3_small(enc.conv_in)
        h = nv.conv3x3_im2col(h, w, b)
        for lvl in range(enc.num_resolutions):
            for rb in enc.down[lvl].block:
                h = run_vae_resnet(rb, h)
            if lvl != enc.num_resolutions - 1:
                w, b = pk_conv3(enc.down[lvl].downsample.conv)
                h = nv.conv3x3(h, w, b, stride=2, tap_off=1)
        h = run_vae_resnet(enc.mid.block_1, h)
        h = run_vae_attn(enc.mid.attn_1, h)
        h = run_vae_resnet(enc.mid.block_2, h)
        g, b = pk_norm(enc.norm_out)
        h = nv.groupnorm(h, g, b, enc.norm_out.eps, silu=True)
        w, b = pk_conv3(enc.conv_out)                                      # [2*zc -> 8 rows]
        h = nv.conv3x3(h, w, b)
        wq, bq = pk_lin(self.quant_conv)
        mom = nv.conv1x1(h, wq, bq)                                        # [B,h,w,8]: mean | logvar
        zc = self.quant_conv.weight.shape[0] // 2
        if out_posterior:
            return DiagonalGaussianDistribution(mom, zc)
        noise = torch.randn((B, zc, mom.shape[1], mom.shape[2])).to(mom.device)   # distributions.py:36
        return nv.vae_posterior(mom, zc, noise=noise, scale=post_scale, want=("sample",))["sample"]

    @torch.no_grad()
    def decode(self, z: torch.Tensor, pre_scale: float = 1.0) -> torch.Tensor:
        """autokl.py:44-54: post_quant_conv -> Decoder -> (x+1)/2 -> clamp.  z: NCHW latents (already
        divided by the latent scale unless `pre_scale` carries 1/scale).  Returns NCHW fp16 in [0,1]."""
        dec = self.decoder
        B, Cz, H, W = z.shape
        nv.gn_reset()
        zc = nv.nchw_to_nhwc(z if z.dtype == torch.float32 else z.to(torch.float16), cpad=8)
        wq, bq = pk_lin(self.post_quant_conv)                              # [8, 8] zero-padded 4x4
        h = nv.linear(zc.reshape(B * H * W, 8), wq, bq, alpha=pre_scale).reshape(B, H, W, 8)
        w, b = cached_conv_in(dec.conv_in, Cz)
        h = nv.conv3x3_im2col(h, w, b)
        h = run_vae_resnet(dec.mid.block_1, h)
        h = run_vae_attn(dec.mid.attn_1, h)
        h = run_vae_resnet(dec.mid.block_2, h)
        for lvl in reversed(range(dec.num_resolutions)):
            up = dec.up[lvl]
            for rb in up.block:
                h = run_vae_resnet(rb, h)
            if lvl != 0:
                w, b = pk_conv3(up.upsample.conv)
                h = nv.conv3x3(nv.upsample2x(h), w, b)
        g, b = pk_norm(dec.norm_out)
        h = nv.groupnorm(h, g, b, dec.norm_out.eps, silu=True)
        w, b = pk_conv3(dec.conv_out)                                      # rows padded 3 -> 8
        h = nv.conv3x3(h, w, b)
        return nv.nhwc_to_nchw(h, dec.out_ch, mul=0.5, add=0.5, lo=0.0, hi=1.0)

    def forward(self, z):
        return self.decode(z)


class DiagonalGaussianDistribution(object):
    """distributions.py:24-37 over the channel-last moments tensor; fields are NCHW fp16 tensors."""

    def __init__(self, moments: torch.Tensor, zc: int):
        self._mom, self._zc = moments, zc
        o = nv.vae_posterior(moments, zc, want=("mean", "logvar", "std"))
        self.mean, self.logvar, self.std = o["mean"], o["logvar"], o["std"]
        self.deterministic = False

    def sample(self):
        noise = torch.randn(self.mean.shape).to(self.mean.device)        # distributions.py:36
        return nv.vae_posterior(self._mom, self._zc, noise=noise, want=("sample",))["sample"]

    def mode(self):
        return self.mean


def cached_conv_in(conv: Conv2d, cz: int):
    """conv_in consumes the 8-channel (zero-padded) post_quant output: pack [O, 9*8] with zero columns
    for the pad channels so the im2col row (k = tap*8 + c) lines up."""
    from .modules import cached, fp16

    def build():
        o = conv.weight.shape[0]
        w = torch.zeros((o, 3, 3, 8), device=conv.weight.device, dtype=torch.float16)
        w[..., :cz] = fp16(conv.weight).permute(0, 2, 3, 1)
        return w.reshape(o, 72).contiguous(), fp16(conv.bias)
    return cached(conv, "conv_in8", [conv.weight, conv.bias], build)
