"""SD-v1.5 UNet (UNetModel2D_Next) on the pfd_b200 kernels.

Module tree, constructor arguments and state-dict keys mirror the reference
(lib/model_zoo/openaimodel.py:2575-2812, :162-274; lib/model_zoo/attention.py:44-71,159-201,277-371)
so reference checkpoints load with strict=True; the arithmetic is a channel-last fp16 pipeline of
C-ABI calls:

  ResBlock            = GN+SiLU -> conv3x3(+bias +time-embedding row add) -> GN+SiLU ->
                        conv3x3(+bias, + fused 1x1 skip conv as extra K segments | + identity residual)
  SpatialTransformer  = GN -> proj_in -> [LN -> self-attn -> +x] [LN -> cross-attn -> +x]
                        [LN -> GEGLU GEMM -> out GEMM -> +x] -> proj_out (+x_in), all token-major
                        (no NCHW<->NLC transposes: channel-last pixels *are* tokens)
  skip concat         = never materialised raw: GN reads both sources and the skip conv takes two K segments.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import native as nv
from . import attention as att
from .attention import attend, ceil8, project_heads, project_heads_fused, project_vt_swapped
from .modules import (Conv2d, GroupNorm, IndexedSequential, LayerNorm, Linear, cached, pk_conv3,
                      pk_conv3_small, pk_lin, pk_mat, pk_norm)


# ------------------------------------------------------------------------------------------------
# parameter tree (names identical to the reference)
# ------------------------------------------------------------------------------------------------
class ResBlock(nn.Module):
    """openaimodel.py:162-274 (use_scale_shift_norm=False, no up/down)."""

    def __init__(self, channels, emb_channels, dropout=0.0, out_channels=None, **_):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.in_layers = IndexedSequential(GroupNorm(32, channels), nn.SiLU(),
                                           Conv2d(channels, self.out_channels, 3, padding=1))
        self.emb_layers = IndexedSequential(nn.SiLU(), Linear(emb_channels, self.out_channels))
        self.out_layers = IndexedSequential(GroupNorm(32, self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                            Conv2d(self.out_channels, self.out_channels, 3, padding=1))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = Conv2d(channels, self.out_channels, 1)


class Downsample(nn.Module):
    """openaimodel.py:133-159 (use_conv=True): 3x3 stride-2 conv."""

    def __init__(self, channels, out_channels=None):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.op = Conv2d(channels, self.out_channels, 3, stride=2, padding=1)


class Upsample(nn.Module):
    """openaimodel.py:89-117 (use_conv=True): nearest 2x + 3x3 conv."""

    def __init__(self, channels, out_channels=None):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.conv = Conv2d(channels, self.out_channels, 3, padding=1)


class CrossAttention(nn.Module):
    """attention.py:159-176."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = context_dim or query_dim
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.to_q = Linear(query_dim, inner, bias=False)
        self.to_k = Linear(context_dim, inner, bias=False)
        self.to_v = Linear(context_dim, inner, bias=False)
        self.to_out = IndexedSequential(Linear(inner, query_dim), nn.Dropout(dropout))


class GEGLU(nn.Module):
    """attention.py:44-51."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    """attention.py:54-71 (glu=True)."""

    def __init__(self, dim, mult=4, dropout=0.0):
        super().__init__()
        inner = int(dim * mult)
        self.net = IndexedSequential(GEGLU(dim, inner), nn.Dropout(dropout), Linear(inner, dim))


class BasicTransformerBlock(nn.Module):
    """attention.py:277-306."""

    def __init__(self, dim, n_heads, d_head, context_dim=None):
        super().__init__()
        self.attn1 = CrossAttention(dim, None, n_heads, d_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, context_dim, n_heads, d_head)
        self.norm1 = LayerNorm(dim)
        self.norm2 = LayerNorm(dim)
        self.norm3 = LayerNorm(dim)


class SpatialTransformer(nn.Module):
    """attention.py:309-371 (use_linear=False, depth=1)."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, context_dim=None, **_):
        super().__init__()
        if isinstance(context_dim, (list, tuple)):
            context_dim = context_dim[0]
        inner = n_heads * d_head
        self.in_channels = in_channels
        self.n_heads, self.d_head = n_heads, d_head
        self.norm = GroupNorm(32, in_channels, eps=1e-6)
        self.proj_in = Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, n_heads, d_head, context_dim) for _ in range(depth)])
        self.proj_out = Conv2d(inner, in_channels, 1)


# ------------------------------------------------------------------------------------------------
# executors
# ------------------------------------------------------------------------------------------------
def run_resblock(rb: ResBlock, x: torch.Tensor, x2: Optional[torch.Tensor], emb_out: torch.Tensor) -> torch.Tensor:
    """x (and optional concat partner x2): channel-last [B,H,W,C]; emb_out: [B, Cout] rows (may be a
    column slice of the batched emb GEMM output)."""
    n0, n1 = rb.in_layers[0], rb.out_layers[0]
    g, b = pk_norm(n0)
    h = nv.groupnorm(x, g, b, n0.eps, silu=True, x2=x2)
    w1, b1 = pk_conv3(rb.in_layers[2])
    h = nv.conv3x3(h, w1, b1, rowadd=emb_out)
    g, b = pk_norm(n1)
    h = nv.groupnorm(h, g, b, n1.eps, silu=True)
    if isinstance(rb.skip_connection, nn.Identity):
        w2, b2 = pk_conv3(rb.out_layers[3])
        return nv.conv3x3(h, w2, b2, residual=x)
    w2, b2 = pk_conv3(rb.out_layers[3], rb.skip_connection)
    return nv.conv3x3(h, w2, b2, skip=[x] if x2 is None else [x, x2])


def _cat_weights(owner: nn.Module, key: str, lins) -> torch.Tensor:
    """Row-concatenated fp16 weights of bias-free Linear layers (fused q|k|v / k|v projection)."""
    return cached(owner, key, [l.weight for l in lins],
                  lambda: torch.cat([l.weight.detach().half() for l in lins], 0).contiguous())


def context_kv(st: SpatialTransformer, context: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """to_k / to_v of the cross-attention for a context [Bc, Nk, Cctx]; constant across DDIM steps."""
    blk = st.transformer_blocks[0]
    Bc, Nk, Cc = context.shape
    ctx2d = context.reshape(Bc * Nk, Cc)
    wk, _ = pk_lin(blk.attn2.to_k)
    wv, _ = pk_lin(blk.attn2.to_v)
    k = project_heads(ctx2d, wk, None, Bc, Nk, st.n_heads, st.d_head)
    vt = project_heads(ctx2d, wv, None, Bc, Nk, st.n_heads, st.d_head, transposed=True)
    return k, vt


def run_spatial_transformer(st: SpatialTransformer, x: torch.Tensor, context: torch.Tensor,
                            kv: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
    B, H, W, C = x.shape
    N = H * W
    heads, d = st.n_heads, st.d_head
    blk = st.transformer_blocks[0]
    g, b = pk_norm(st.norm)
    xn = nv.groupnorm(x, g, b, st.norm.eps, silu=False)
    w, bb = pk_lin(st.proj_in)
    t = nv.linear(xn.reshape(B * N, C), w, bb)                                  # [B*N, inner]
    inner = t.shape[1]
    # --- self attention (attention.py:303)
    g, b = pk_norm(blk.norm1)
    n1 = nv.layernorm(t, g, b, blk.norm1.eps)
    a = blk.attn1
    if att.USE_FUSED_QK and N % 8 == 0:
        qk = project_heads_fused(n1, _cat_weights(a, "qk_cat", [a.to_q, a.to_k]), None, B, N, heads, d, 2)
        vt4 = project_vt_swapped(n1, pk_lin(a.to_v)[0], B, N, heads, d)
        o = nv.flash_attn_strided(qk[:, :heads], qk[:, heads:], vt4, Nq=N, Nk=N, scale=a.scale,
                                  out=torch.empty((B, N, inner), device=t.device, dtype=torch.float16))
    else:
        q = project_heads(n1, pk_lin(a.to_q)[0], None, B, N, heads, d)
        k = project_heads(n1, pk_lin(a.to_k)[0], None, B, N, heads, d)
        vt = project_heads(n1, pk_lin(a.to_v)[0], None, B, N, heads, d, transposed=True)
        o = attend(q, k, vt, B=B, heads=heads, Nq=N, Nk=N, scale=a.scale)
    w, bb = pk_lin(a.to_out[0])
    t = nv.linear(o.reshape(B * N, inner), w, bb, residual=t)
    # --- cross attention (attention.py:304)
    g, b = pk_norm(blk.norm2)
    n2 = nv.layernorm(t, g, b, blk.norm2.eps)
    a = blk.attn2
    if kv is None:
        kv = context_kv(st, context)
    q = project_heads(n2, pk_lin(a.to_q)[0], None, B, N, heads, d)
    o = attend(q, kv[0], kv[1], B=B, heads=heads, Nq=N, Nk=context.shape[1], scale=a.scale)
    w, bb = pk_lin(a.to_out[0])
    t = nv.linear(o.reshape(B * N, inner), w, bb, residual=t)
    # --- GEGLU feed-forward (attention.py:305)
    g, b = pk_norm(blk.norm3)
    n3 = nv.layernorm(t, g, b, blk.norm3.eps)
    proj = blk.ff.net[0].proj
    wg, bg, bn = cached(proj, "geglu", [proj.weight, proj.bias],
                        lambda: nv.pack_geglu(proj.weight.detach().half().contiguous(),
                                              proj.bias.detach().half().contiguous()))
    gg = nv.linear(n3, wg, bg, act=nv.ACT_GEGLU, bn_force=bn)
    w, bb = pk_lin(blk.ff.net[2])
    t = nv.linear(gg, w, bb, residual=t)
    # --- proj_out + residual with the block input (attention.py:368-371)
    w, bb = pk_lin(st.proj_out)
    out = nv.linear(t, w, bb, residual=x.reshape(B * N, C))
    return out.reshape(B, H, W, C)


def time_embed_silu(time_embed: IndexedSequential, t: torch.Tensor, model_channels: int) -> torch.Tensor:
    """silu(time_embed(timestep_embedding(t))) — every consumer (ResBlock.emb_layers, openaimodel.py:217)
    applies SiLU first, so it is fused into the second GEMM's epilogue."""
    te = nv.timestep_embedding(t, model_channels)
    w0, b0 = pk_lin(time_embed[0])
    w2, b2 = pk_lin(time_embed[2])
    e = nv.linear(te, w0, b0, act=nv.ACT_SILU)
    return nv.linear(e, w2, b2, act=nv.ACT_SILU)


def batched_emb_layers(owner: nn.Module, resblocks: Sequence[ResBlock], silu_emb: torch.Tensor) -> List[torch.Tensor]:
    """All ResBlock.emb_layers Linear layers as ONE GEMM; returns per-block [B, Cout] column slices."""
    lins = [rb.emb_layers[1] for rb in resblocks]
    params = [p for l in lins for p in (l.weight, l.bias)]

    def build():
        w = torch.cat([l.weight.detach().half() for l in lins], 0).contiguous()
        b = torch.cat([l.bias.detach().half() for l in lins], 0).contiguous()
        return w, b
    w, b = cached(owner, "emb_cat", params, build)
    out = nv.linear(silu_emb, w, b)
    res, off = [], 0
    for l in lins:
        n = l.weight.shape[0]
        res.append(out[:, off:off + n])
        off += n
    return res


# ------------------------------------------------------------------------------------------------
class UNetModel2D_Next(nn.Module):
    """openaimodel.py:2575-2812 — same constructor arguments, buffers and layer orders."""

    def __init__(self, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 context_dim, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, use_checkpoint=False,
                 num_heads=8, num_head_channels=None, parts=('global', 'data', 'context')):
        super().__init__()
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        if isinstance(num_res_blocks, int):
            num_res_blocks = len(channel_mult) * [num_res_blocks]
        self.num_res_blocks = list(num_res_blocks)
        self.attention_resolutions = list(attention_resolutions)
        self.context_dim, self.dropout = context_dim, dropout
        self.channel_mult = list(channel_mult)
        self.num_heads, self.num_head_channels = num_heads, num_head_channels
        self.parts = list(parts) if isinstance(parts, (list, tuple)) else [parts]
        assert all(p in self.parts for p in ('global', 'data', 'context')), \
            "pfd_b200 builds the complete UNet (parts: global, data, context)"
        ted = model_channels * 4
        self.time_embed = IndexedSequential(Linear(model_channels, ted), nn.SiLU(), Linear(ted, ted))
        self.data_blocks = nn.ModuleList([])
        self.context_blocks = nn.ModuleList([])
        order: List[str] = []

        def add_d(layer):
            self.data_blocks.append(IndexedSequential(layer))
            order.append('d')

        def add_c(ch):
            d_head, n_heads = self.get_d_head_n_heads(ch)
            self.context_blocks.append(IndexedSequential(
                SpatialTransformer(ch, n_heads, d_head, context_dim=context_dim)))
            order.append('c')

        add_d(Conv2d(in_channels, model_channels, 3, padding=1))
        order.append('save_hidden_feature')
        chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(channel_mult):
            for _ in range(self.num_res_blocks[level]):
                add_d(ResBlock(ch, ted, dropout, out_channels=mult * model_channels))
                ch = mult * model_channels
                if ds in attention_resolutions:
                    add_c(ch)
                chans.append(ch)
                order.append('save_hidden_feature')
            if level != len(channel_mult) - 1:
                add_d(Downsample(ch, out_channels=ch))
                chans.append(ch)
                order.append('save_hidden_feature')
                ds *= 2
        self.i_order = list(order)
        order.clear()
        add_d(ResBlock(ch, ted, dropout))
        add_c(ch)
        add_d(ResBlock(ch, ted, dropout))
        self.m_order = list(order)
        order.clear()
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for _ in range(self.num_res_blocks[level] + 1):
                order.append('load_hidden_feature')
                ich = chans.pop()
                add_d(ResBlock(ch + ich, ted, dropout, out_channels=model_channels * mult))
                ch = model_channels * mult
                if ds in attention_resolutions:
                    add_c(ch)
            if level != 0:
                add_d(Upsample(ch, out_channels=ch))
                ds //= 2
        add_d(IndexedSequential(GroupNorm(32, ch), nn.SiLU(), Conv2d(model_channels, out_channels, 3, padding=1)))
        self.o_order = list(order)
        self.layer_order = self.i_order + self.m_order + self.o_order
        self.parameter_group = {'global': self.time_embed, 'data': self.data_blocks,
                                'context': self.context_blocks}

    def get_d_head_n_heads(self, ch):
        if self.num_head_channels is None:
            return ch // self.num_heads, self.num_heads
        return self.num_head_channels, ch // self.num_head_channels

    # -------------------------------------------------------------------------------------------
    def resblocks(self) -> List[ResBlock]:
        return [blk[0] for blk in self.data_blocks if isinstance(blk[0], ResBlock)]

    def prepare_context(self, context: torch.Tensor) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """Cross-attention K / V^T of every context block for a fixed context (reused for all steps)."""
        return [context_kv(cb[0], context) for cb in self.context_blocks]

    def run_data_block(self, idx: int, h, h2, embs: Dict[int, torch.Tensor]):
        layer = self.data_blocks[idx][0]
        if isinstance(layer, ResBlock):
            return run_resblock(layer, h, h2, embs[idx])
        assert h2 is None
        if isinstance(layer, Downsample):
            w, b = pk_conv3(layer.op)
            return nv.conv3x3(h, w, b, stride=2)
        if isinstance(layer, Upsample):
            w, b = pk_conv3(layer.conv)
            return nv.conv3x3(nv.upsample2x(h), w, b)
        if isinstance(layer, IndexedSequential):                      # GN, SiLU, conv (openaimodel.py:2732)
            g, b = pk_norm(layer[0])
            hn = nv.groupnorm(h, g, b, layer[0].eps, silu=True)
            w, bb = pk_conv3(layer[2])                                # rows padded to 8 output channels
            return nv.conv3x3(hn, w, bb)
        if isinstance(layer, Conv2d):                                 # stem conv, Cin=4: im2col path
            w, b = pk_conv3_small(layer)
            return nv.conv3x3_im2col(h, w, b)
        raise RuntimeError(f"unknown data block {type(layer)}")

    def apply(self, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor,
              control: Optional[List[torch.Tensor]] = None,
              kv: Optional[List[Tuple[torch.Tensor, torch.Tensor]]] = None,
              mixed_contexts: Optional[List[Tuple[torch.Tensor, float]]] = None) -> torch.Tensor:
        """pfd.py:314-365 / 466-528.  x: NCHW latents, context [B, Nk, Cctx], control: ControlNet
        residuals as channel-last tensors (list of 13, consumed from the end).  Returns NCHW fp16.
        mixed_contexts: [(context, ratio)] — pfd.py:367-439 `apply_model_multicontext` ('attention' mixing): every
        context block becomes sum_i ratio_i * block(h, context_i)."""
        x = x.to(torch.float16)
        context = context.to(torch.float16).contiguous()
        B = x.shape[0]
        nv.gn_reset()
        silu_emb = time_embed_silu(self.time_embed, timesteps, self.model_channels)
        rbs = [i for i, blk in enumerate(self.data_blocks) if isinstance(blk[0], ResBlock)]
        emb_list = batched_emb_layers(self, [self.data_blocks[i][0] for i in rbs], silu_emb)
        embs = dict(zip(rbs, emb_list))
        if kv is None and mixed_contexts is None:
            kv = self.prepare_context(context)
        ccs = list(control) if control is not None else None
        h = nv.nchw_to_nhwc(x)
        h2 = None
        hs: List[torch.Tensor] = []
        di = ci = 0
        for lt in self.i_order + self.m_order + ['__mid__'] + self.o_order:
            if lt == 'd':
                h = self.run_data_block(di, h, h2, embs)
                h2 = None
                di += 1
            elif lt == 'c':
                st = self.context_blocks[ci][0]
                if mixed_contexts is None:
                    h = run_spatial_transformer(st, h, context, kv[ci])
                else:                                                    # pfd.py:374-379 context_mixing
                    acc = None
                    for cm, r in mixed_contexts:
                        hi = run_spatial_transformer(st, h, cm.to(torch.float16).contiguous(), None)
                        acc = nv.axpby(hi, r) if acc is None else nv.axpby(acc, 1.0, hi, r)
                    h = acc
                ci += 1
            elif lt == 'save_hidden_feature':
                hs.append(h)
            elif lt == '__mid__':
                if ccs is not None:
                    h = nv.axpby(h, 1.0, ccs.pop(), 1.0)                 # pfd.py:515
            elif lt == 'load_hidden_feature':
                h2 = hs.pop()
                if ccs is not None:
                    h2 = nv.axpby(h2, 1.0, ccs.pop(), 1.0)               # pfd.py:519
        return nv.nhwc_to_nchw(h, self.out_channels)

    def forward(self, x, timesteps, context):
        return self.apply(x, timesteps, context)
