"""Diffuser UNet of Versatile Diffusion on vdb200 kernels: ResBlock / Downsample / Upsample /
UNetModel2D_Next (+ the context-block half of UNetModel0D_Next).
Reference: lib/model_zoo/openaimodel.py:72-274 (blocks), :2575-2812 (UNetModel2D_Next), :2814-2975
(UNetModel0D_Next).  Same constructor signatures, attribute names (data_blocks, context_blocks,
time_embed, i_order/m_order/o_order/layer_order, parameter_group) and state_dict keys.

Data layout: blocks exchange NHWC bf16 activations; a block input may be a PAIR (h, skip) standing for
torch.cat([h, hs.pop()], dim=1) of the reference (vd.py:372) — the concat is never materialised: the
GroupNorm kernel reads both halves, and the 1x1 skip_connection runs as extra K segments of conv2.

Kernel schedule of a ResBlock (reference _forward, :254-274):
  GN32+SiLU (2 kernels) -> conv3x3 [+ emb_out + bias in the epilogue] -> GN32+SiLU -> conv3x3
  [+ 1x1 skip over the raw input as K segments | + identity residual] ; emb_layers of ALL ResBlocks
  are evaluated by one skinny GEMM per UNet call (UNetModel2D_Next.embed_all).
"""
import copy
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from lib.model_zoo.common.get_model import register
from .attention import SpatialTransformer
from .diffusion_utils import (PackedMixin, PackedModule, bf16, f32, conv_nd, linear, normalization, pack_conv1x1, pack_conv3x3,
                              require_cuda, timestep_embedding, zero_module, fold_upsample_conv3x3,
                              upsample_fold_enabled)  # noqa: F401


def _ops():
    from vdb200 import ops
    return ops


def _first(x):
    return x[0] if isinstance(x, tuple) else x


class TimestepBlock(nn.Module):
    """Marker: forward(x, emb)."""


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """Passes emb / context to the children that take them (reference :72-86)."""

    def forward(self, x, emb, context=None):
        for layer in self:
            if isinstance(layer, TimestepBlock):
                x = layer(x, emb)
            elif isinstance(layer, SpatialTransformer):
                x = layer(x, context)
            else:
                x = layer(x)
        return x


class Upsample(PackedModule):
    """nearest 2x + 3x3 conv (reference :89-117)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if use_conv:
            self.conv = conv_nd(dims, self.channels, self.out_channels, 3, padding=padding)

    def _pack(self):
        if not self.use_conv:
            return {}
        d = {"w": pack_conv3x3(self.conv.weight), "b": f32(self.conv.bias)}
        if upsample_fold_enabled(1 << 30, self.out_channels):   # (the folded copy is only built when some input can use it)
            d["wf"] = fold_upsample_conv3x3(self.conv.weight)
        return d

    def forward(self, x):
        ops = _ops()
        require_cuda(x, "Upsample")
        if self.use_conv and upsample_fold_enabled(x.shape[0] * x.shape[1] * x.shape[2], self.out_channels):
            p = self.packed()
            return ops.upsample2x_conv3x3_folded(x, p["wf"], bias=p["b"])     # 2.25x fewer FLOPs, no upsampled temporary
        x = ops.upsample2x(x)
        if self.use_conv:
            p = self.packed()
            x = ops.conv3x3(x, p["w"], bias=p["b"])
        return x


class Downsample(PackedModule):
    """3x3 stride-2 pad-1 conv (reference :133-159)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if not use_conv:
            raise NotImplementedError("avg-pool Downsample is not used by the VD configs")
        self.op = conv_nd(dims, self.channels, self.out_channels, 3, stride=2, padding=padding)

    def _pack(self):
        return {"w": pack_conv3x3(self.op.weight), "b": f32(self.op.bias)}

    def forward(self, x):
        require_cuda(x, "Downsample")
        p = self.packed()
        return _ops().conv3x3(x, p["w"], bias=p["b"], mode=1)


class ResBlock(PackedModule, TimestepBlock):
    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False,
                 use_scale_shift_norm=False, dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        if use_scale_shift_norm or up or down or use_conv:
            raise NotImplementedError("VD uses ResBlock(use_scale_shift_norm=False, up=False, down=False, use_conv=False)")
        self.channels = channels
        self.emb_channels = emb_channels
        self.dropout = dropout
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.use_checkpoint = use_checkpoint
        self.use_scale_shift_norm = use_scale_shift_norm
        self.updown = False
        self.in_layers = nn.Sequential(normalization(channels), nn.SiLU(),
                                       conv_nd(dims, channels, self.out_channels, 3, padding=1))
        self.h_upd = self.x_upd = nn.Identity()
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(conv_nd(dims, self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = conv_nd(dims, channels, self.out_channels, 1)
        self.emb_slot = None  # (offset, total) into the UNet-level fused emb projection, set by the owner

    def _pack(self):
        w2 = pack_conv3x3(self.out_layers[3].weight)
        b2 = f32(self.out_layers[3].bias)
        has_skip = not isinstance(self.skip_connection, nn.Identity)
        if has_skip:
            w2 = torch.cat([w2, pack_conv1x1(self.skip_connection.weight)], dim=1).contiguous()
            b2 = (b2 + f32(self.skip_connection.bias)).contiguous()
        return {"g1": f32(self.in_layers[0].weight), "be1": f32(self.in_layers[0].bias),
                "w1": pack_conv3x3(self.in_layers[2].weight), "b1": f32(self.in_layers[2].bias),
                "we": bf16(self.emb_layers[1].weight), "bemb": f32(self.emb_layers[1].bias),
                "g2": f32(self.out_layers[0].weight), "be2": f32(self.out_layers[0].bias),
                "w2": w2, "b2": b2, "has_skip": has_skip}

    def forward(self, x, emb):
        """x: NHWC bf16 [B,H,W,C] or a pair (h, skip) == cat along C.
        emb: either the [B, emb_channels] fp32 time embedding (stand-alone use) or an EmbTable produced by
        UNetModel2D_Next.embed_all (emb_out + conv1 bias for every ResBlock, one kernel)."""
        ops = _ops()
        p = self.packed()
        x1, x2 = x if isinstance(x, tuple) else (x, None)
        require_cuda(x1, "ResBlock")
        eps = self.in_layers[0].eps
        a1 = ops.groupnorm(x1, p["g1"], p["be1"], eps, act=ops.ACT_SILU, x2=x2)
        if isinstance(emb, EmbTable):
            bias1, bstride = emb.slot(self.emb_slot[0]), emb.total
        else:
            bias1 = ops.linear_small(emb.float().contiguous(), p["we"], (p["bemb"] + p["b1"]).contiguous(), act_in=ops.ACT_SILU)
            bstride = self.out_channels
        h = ops.conv3x3(a1, p["w1"], bias=bias1, bias_bstride=bstride)
        a2 = ops.groupnorm(h, p["g2"], p["be2"], self.out_layers[0].eps, act=ops.ACT_SILU)
        if p["has_skip"]:
            return ops.conv3x3(a2, p["w2"], bias=p["b2"], skip1=x1, skip2=x2)
        return ops.conv3x3(a2, p["w2"], bias=p["b2"], resid=x1)


class EmbTable(object):
    """[B, total] fp32: SiLU(emb) @ We^T + be + b_conv1 for every ResBlock of the UNet (column slices)."""

    def __init__(self, table):
        self.table = table
        self.total = table.shape[1]

    def slot(self, offset):
        return self.table.view(-1)[offset:]


class OutHead(PackedModule):
    """GroupNorm -> SiLU -> conv3x3(model_channels -> out_channels) (reference :2732-2737).
    Registered under the reference's Sequential indices 0 (norm) and 2 (conv)."""

    def __init__(self, ch, model_channels, out_channels):
        super().__init__()
        self.add_module("0", normalization(ch))
        self.add_module("1", nn.SiLU())
        self.add_module("2", zero_module(conv_nd(2, model_channels, out_channels, 3, padding=1)))

    def _pack(self):
        norm, conv = getattr(self, "0"), getattr(self, "2")
        return {"g": f32(norm.weight), "b": f32(norm.bias), "w": pack_conv3x3(conv.weight), "bc": f32(conv.bias)}

    def forward(self, x):
        ops = _ops()
        p = self.packed()
        a = ops.groupnorm(x, p["g"], p["b"], getattr(self, "0").eps, act=ops.ACT_SILU)
        return ops.conv3x3(a, p["w"], bias=p["bc"], out_dtype=torch.float32)   # NHWC fp32 [B,H,W,out]


class ConvIn(PackedMixin, nn.Conv2d):
    """conv3x3(in_channels=4 -> model_channels) on the fp32 NHWC latent: im2col (K = 36 -> 64) + GEMM.
    Subclasses nn.Conv2d so the checkpoint keys stay `data_blocks.0.0.{weight,bias}` (reference :2664)."""

    def __init__(self, in_channels, model_channels):
        super().__init__(in_channels, model_channels, 3, padding=1)

    def _pack(self):
        w = self.weight.detach()
        n, cin = w.shape[0], w.shape[1]
        kpad = 64
        wp = torch.zeros(n, kpad, dtype=torch.bfloat16, device=w.device)
        wp[:, :9 * cin] = w.permute(0, 2, 3, 1).reshape(n, -1).to(torch.bfloat16)
        return {"w": wp, "b": f32(self.bias), "kpad": kpad}

    def forward(self, x):  # x: fp32 NHWC [B,H,W,Cin]
        ops = _ops()
        p = self.packed()
        B, H, W, _ = x.shape
        col = ops.im2col3x3_small(x, kpad=p["kpad"])
        return ops.gemm(col, p["w"], bias=p["b"]).view(B, H, W, -1)


@register('openai_unet_2d_next')
class UNetModel2D_Next(nn.Module):
    def __init__(self, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 context_dim, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, use_checkpoint=False,
                 num_heads=8, num_head_channels=None, parts=['global', 'data', 'context']):
        super().__init__()
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        if isinstance(num_res_blocks, int):
            self.num_res_blocks = len(channel_mult) * [num_res_blocks]
        else:
            if len(num_res_blocks) != len(channel_mult):
                raise ValueError("provide num_res_blocks either as an int (globally constant) or "
                                 "as a list/tuple (per-level) with the same length as channel_mult")
            self.num_res_blocks = list(num_res_blocks)
        self.attention_resolutions = attention_resolutions
        self.context_dim = context_dim
        self.dropout = dropout
        self.channel_mult = channel_mult
        self.conv_resample = conv_resample
        self.use_checkpoint = use_checkpoint   # accepted for config compatibility; sampling never checkpoints
        self.num_heads = num_heads
        self.num_head_channels = num_head_channels
        assert (num_heads is None) + (num_head_channels is None) == 1, \
            "One of num_heads or num_head_channels need to be set"
        self.parts = parts if isinstance(parts, list) else [parts]
        self.glayer_included = 'global' in self.parts
        self.dlayer_included = 'data' in self.parts
        self.clayer_included = 'context' in self.parts
        self.layer_sequence_ordering = []

        time_embed_dim = model_channels * 4
        if self.glayer_included:
            self.time_embed = nn.Sequential(linear(model_channels, time_embed_dim), nn.SiLU(),
                                            linear(time_embed_dim, time_embed_dim))
        if self.dlayer_included:
            self.data_blocks = nn.ModuleList([])
            ResBlockDefault = partial(ResBlock, emb_channels=time_embed_dim, dropout=dropout, dims=2,
                                      use_checkpoint=use_checkpoint, use_scale_shift_norm=False)
        else:
            ResBlockDefault = lambda *a, **k: None
        if self.clayer_included:
            self.context_blocks = nn.ModuleList([])
            CrossAttnDefault = partial(SpatialTransformer, context_dim=context_dim, disable_self_attn=False)
        else:
            CrossAttnDefault = lambda *a, **k: None

        self.add_data_layer(ConvIn(in_channels, model_channels) if self.dlayer_included else None)
        self.layer_sequence_ordering.append('save_hidden_feature')
        input_block_chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(channel_mult):
            for _ in range(self.num_res_blocks[level]):
                self.add_data_layer(ResBlockDefault(channels=ch, out_channels=mult * model_channels))
                ch = mult * model_channels
                if ds in attention_resolutions:
                    d_head, n_heads = self.get_d_head_n_heads(ch)
                    self.add_context_layer(CrossAttnDefault(in_channels=ch, d_head=d_head, n_heads=n_heads))
                input_block_chans.append(ch)
                self.layer_sequence_ordering.append('save_hidden_feature')
            if level != len(channel_mult) - 1:
                self.add_data_layer(Downsample(ch, use_conv=True, dims=2, out_channels=ch) if self.dlayer_included else None)
                input_block_chans.append(ch)
                self.layer_sequence_ordering.append('save_hidden_feature')
                ds *= 2
        self.i_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_sequence_ordering = []

        self.add_data_layer(ResBlockDefault(channels=ch))
        d_head, n_heads = self.get_d_head_n_heads(ch)
        self.add_context_layer(CrossAttnDefault(in_channels=ch, d_head=d_head, n_heads=n_heads))
        self.add_data_layer(ResBlockDefault(channels=ch))
        self.m_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_sequence_ordering = []

        for level, mult in list(enumerate(channel_mult))[::-1]:
            for _ in range(self.num_res_blocks[level] + 1):
                self.layer_sequence_ordering.append('load_hidden_feature')
                ich = input_block_chans.pop()
                self.add_data_layer(ResBlockDefault(channels=ch + ich, out_channels=model_channels * mult))
                ch = model_channels * mult
                if ds in attention_resolutions:
                    d_head, n_heads = self.get_d_head_n_heads(ch)
                    self.add_context_layer(CrossAttnDefault(in_channels=ch, d_head=d_head, n_heads=n_heads))
            if level != 0:
                self.add_data_layer(Upsample(ch, conv_resample, dims=2, out_channels=ch) if self.dlayer_included else None)
                ds //= 2
        self.add_data_layer(OutHead(ch, model_channels, out_channels) if self.dlayer_included else None)
        self.o_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_order = copy.deepcopy(self.i_order + self.m_order + self.o_order)
        del self.layer_sequence_ordering

        self.parameter_group = {}
        if self.glayer_included:
            self.parameter_group['global'] = self.time_embed
        if self.dlayer_included:
            self.parameter_group['data'] = self.data_blocks
        if self.clayer_included:
            self.parameter_group['context'] = self.context_blocks
        self._emb_packed = None
        self._assign_emb_slots()

    # ------------------------------------------------------------------ construction helpers
    def get_d_head_n_heads(self, ch):
        if self.num_head_channels is None:
            return ch // self.num_heads, self.num_heads
        return self.num_head_channels, ch // self.num_head_channels

    def add_data_layer(self, layer):
        if self.dlayer_included:
            # ConvIn / OutHead stand in for the reference's bare conv / Sequential and expose the same
            # keys (`data_blocks.<i>.0.weight`, `data_blocks.<i>.0.{0,2}.weight`)
            self.data_blocks.append(TimestepEmbedSequential(layer))
        self.layer_sequence_ordering.append('d')

    def add_context_layer(self, layer):
        if self.clayer_included:
            self.context_blocks.append(TimestepEmbedSequential(layer))
        self.layer_sequence_ordering.append('c')

    def _assign_emb_slots(self):
        if not self.dlayer_included:
            return
        off = 0
        for blk in self.data_blocks:
            for layer in blk:
                if isinstance(layer, ResBlock):
                    layer.emb_slot = (off, None)
                    off += layer.out_channels
        self._emb_total = off

    def _apply(self, fn, *a, **k):
        self._emb_packed = self._te_packed = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._emb_packed = self._te_packed = None
        return super()._load_from_state_dict(*a, **k)

    # ------------------------------------------------------------------ fused embedding path
    def _pack_emb(self):
        if self._emb_packed is None:
            with torch.no_grad():
                ws, bs = [], []
                for blk in self.data_blocks:
                    for layer in blk:
                        if isinstance(layer, ResBlock):
                            ws.append(bf16(layer.emb_layers[1].weight))
                            bs.append(f32(layer.emb_layers[1].bias) + f32(layer.in_layers[2].bias))
                self._emb_packed = {"w": torch.cat(ws, 0).contiguous(), "b": torch.cat(bs, 0).contiguous()}
        return self._emb_packed

    def time_embedding(self, t_emb):
        """time_embed MLP (reference :2629-2633) on the fp32 sinusoid [B, model_channels], B <= 16 per call."""
        ops = _ops()
        te = self.time_embed
        w0, b0, w2, b2 = self.time_embed_packed()
        outs = []
        for i in range(0, t_emb.shape[0], 16):
            h = ops.linear_small(t_emb[i:i + 16].contiguous(), w0, b0, act_out=ops.ACT_SILU)
            outs.append(ops.linear_small(h, w2, b2))
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def time_embed_packed(self):
        te = self.time_embed
        if getattr(self, "_te_packed", None) is None:
            self._te_packed = (bf16(te[0].weight), f32(te[0].bias), bf16(te[2].weight), f32(te[2].bias))
        return self._te_packed

    def embed_table(self, t_emb, time_owner=None):
        """Sinusoid [B, model_channels] fp32 -> EmbTable, on the tensor-core GEMM: time_embed MLP (SiLU fused into both
        epilogues: only SiLU(emb) is ever consumed, openaimodel.py:217-223) then ALL ResBlock emb projections as one
        [B, sum(Cout)] GEMM with the conv1 biases folded in.  (The skinny CUDA-core linear took 230 us per step here.)"""
        ops = _ops()
        w0, b0, w2, b2 = (time_owner or self).time_embed_packed()
        p = self._pack_emb()
        h = ops.gemm(ops.to_bf16(t_emb.contiguous()), w0, bias=b0, act=ops.ACT_SILU, ksplit=1)
        s = ops.gemm(h, w2, bias=b2, act=ops.ACT_SILU, ksplit=1)          # SiLU(time_embed(t_emb)), bf16
        return EmbTable(ops.gemm(s, p["w"], bias=p["b"], out_dtype=torch.float32, ksplit=1))

    def embed_all(self, emb):
        """emb [B, 4*model_channels] fp32 -> EmbTable with every ResBlock's SiLU->Linear (+conv1 bias)."""
        ops = _ops()
        p = self._pack_emb()
        outs = [ops.linear_small(emb[i:i + 16].contiguous(), p["w"], p["b"], act_in=ops.ACT_SILU)
                for i in range(0, emb.shape[0], 16)]
        return EmbTable(outs[0] if len(outs) == 1 else torch.cat(outs, 0))

    # ------------------------------------------------------------------ public forward
    def forward(self, x, timesteps, context):
        """x [B,in_channels,H,W] (any float dtype, CUDA), timesteps [B], context [B,L,context_dim] -> eps, same
        shape/dtype as x.  (The reference's forward walks i_order twice — a bug, openaimodel.py:2801 — this one
        walks i/m/o_order as VD_v2_0.apply_model does.)"""
        require_cuda(x, "UNetModel2D_Next")
        ops = _ops()
        xh = ops.nchw_to_nhwc(x.float().contiguous())
        t_emb = timestep_embedding(timesteps, self.model_channels)
        emb = self.embed_table(t_emb)
        h = unet_walk(self, [self], xh, emb, [context], [1.0])
        return ops.nhwc_to_nchw(h).to(x.dtype)


def unet_walk(data_unet, ctx_unets, h, emb, contexts, ratios, key_mass=None):
    """The i/m/o_order walk of VD_v2_0.apply_model / apply_model_multicontext (vd.py:344-381, 404-455):
    'd' blocks from data_unet.data_blocks, 'c' blocks from each ctx_unet.context_blocks mixed by ratio.  key_mass: an
    attention.KeyMass that the mid block's self-attention (the 'c' of m_order) adds its key mass to, each context's at its ratio."""
    hs = []
    d_iter = iter(data_unet.data_blocks)
    c_iters = [iter(u.context_blocks) for u in ctx_unets]
    tot = float(sum(ratios))
    rs = [float(r) / tot for r in ratios]

    def run_c(h, rec=None):
        mods = [next(ci) for ci in c_iters]
        if len(mods) == 1 and rec is None:
            return mods[0](h, emb, contexts[0])
        # context_mixing 'attention' (vd.py:391-396): sum_i r_i*ST_i(h) with sum r_i = 1 == h + sum_i r_i*delta_i,
        # accumulated in the proj_out epilogues (term 1 starts from h, later terms from the running sum)
        acc = None
        for m, c, r in zip(mods, contexts, rs):
            acc = m[0](h, c, ratio=r, acc=acc, key_mass=None if rec is None else rec.weighted(r))
        return acc

    mid = len(data_unet.i_order)
    for n, ltype in enumerate(data_unet.i_order + data_unet.m_order):
        if ltype == 'd':
            h = next(d_iter)(h, emb, None)
        elif ltype == 'c':
            h = run_c(h, key_mass if n >= mid else None)
        elif ltype == 'save_hidden_feature':
            hs.append(h)
    for ltype in data_unet.o_order:
        if ltype == 'load_hidden_feature':
            h = (h, hs.pop())
        elif ltype == 'd':
            h = next(d_iter)(h, emb, None)
        elif ltype == 'c':
            h = run_c(h)
    return h


def _md_perm(C, sdim, device):
    """Index map between the reference's flattening of a [C, sdim, 1] multi-dim feature (index c*sdim + s, openaimodel.py:2287-2293)
    and this build's NHWC order (index s*C + c): ours[i] = ref[perm[i]]."""
    idx = torch.arange(C * sdim, device=device)
    s, c = idx // C, idx % C
    return c * sdim + s


class Linear_MultiDim(PackedMixin, nn.Linear):
    """nn.Linear over a flattened multi-dim feature (reference openaimodel.py:2275-2293); same parameter names / shapes.
    Here the [B, C, sdim, 1] features of the 0-D diffuser live as NHWC bf16 [B, sdim, 1, C]; the rows / columns of the weight
    are permuted once at pack time so that the GEMM reads and writes that order directly."""

    def __init__(self, in_features, out_features, *args, **kwargs):
        in_features = [in_features] if isinstance(in_features, int) else list(in_features)
        out_features = [out_features] if isinstance(out_features, int) else list(out_features)
        self.in_features_multidim = in_features
        self.out_features_multidim = out_features
        nn.Linear.__init__(self, int(np.prod(in_features)), int(np.prod(out_features)), *args, **kwargs)

    def _pack(self):
        w, b = self.weight.detach(), self.bias.detach()
        if len(self.out_features_multidim) == 3:
            po = _md_perm(self.out_features_multidim[0], self.out_features_multidim[1], w.device)
            w, b = w[po], b[po]
        if len(self.in_features_multidim) == 3:
            pi = _md_perm(self.in_features_multidim[0], self.in_features_multidim[1], w.device)
            w = w[:, pi]
        return {"w": bf16(w), "b": f32(b)}

    def forward(self, x):
        """x: [B, K] (flat input, bf16 or fp32) or NHWC bf16 [B, sdim, 1, C]; returns NHWC bf16 [B, sdim, 1, C] for a
        multi-dim output, fp32 [B, N] for a flat one (the output head)."""
        ops = _ops()
        p = self.packed()
        B = x.shape[0]
        a = x.reshape(B, -1)
        a = a if a.dtype == torch.bfloat16 else ops.to_bf16(a.float().contiguous())
        if len(self.out_features_multidim) == 3:
            C, sdim = self.out_features_multidim[0], self.out_features_multidim[1]
            return ops.gemm(a, p["w"], bias=p["b"]).view(B, sdim, 1, C)
        return ops.gemm(a, p["w"], bias=p["b"], out_dtype=torch.float32)


class FCBlock_MultiDim(PackedModule, TimestepBlock):
    """The 0-D diffuser's residual block (reference FCBlock / FCBlock_MultiDim, openaimodel.py:2084-2141, 2295-2354): the
    [C, sdim, 1] feature flattened to C*sdim channels of a 1x1 image, GroupNorm32 -> SiLU -> 1x1 conv (+ SiLU->Linear(emb)),
    GroupNorm32 -> SiLU -> 1x1 conv, + skip (identity / 1x1 conv).  Parameter names / shapes as in the reference.
    Kernels: GroupNorm over the NHWC [B, sdim, 1, C] view (the reference's 32 groups of the flattened index c*sdim + s are
    exactly 32 channel groups over all sdim positions), the three 1x1 convs as GEMMs over the flattened feature with rows /
    columns permuted to NHWC order; the skip conv runs as extra K columns of the second GEMM.  M = batch rows: these GEMMs
    stream weights (0.2 GB per block at full size) — HBM-bound by construction (SURVEY §8f rank 4)."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_checkpoint=False):
        super().__init__()
        channels = [channels] if isinstance(channels, int) else list(channels)
        self.channels_multidim = channels
        self.out_channels_multidim = channels if out_channels is None else \
            ([out_channels] if isinstance(out_channels, int) else list(out_channels))
        self.channels = int(np.prod(self.channels_multidim))
        self.out_channels = int(np.prod(self.out_channels_multidim))
        self.emb_channels = emb_channels
        self.dropout = dropout
        self.use_checkpoint = use_checkpoint
        self.emb_slot = None  # (offset, total) into the diffuser-level fused emb projection, set by the owner
        self.in_layers = nn.Sequential(normalization(self.channels), nn.SiLU(), nn.Conv2d(self.channels, self.out_channels, 1, padding=0))
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(nn.Conv2d(self.out_channels, self.out_channels, 1, padding=0)))
        if self.out_channels == self.channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = nn.Conv2d(self.channels, self.out_channels, 1, padding=0)

    def _pack(self):
        dev = self.in_layers[2].weight.device
        Cin, sdim = self.channels_multidim[0], self.channels_multidim[1]
        Cout = self.out_channels_multidim[0]
        pi, po = _md_perm(Cin, sdim, dev), _md_perm(Cout, sdim, dev)
        w1 = self.in_layers[2].weight.detach().reshape(self.out_channels, self.channels)[po][:, pi]
        w2 = self.out_layers[3].weight.detach().reshape(self.out_channels, self.out_channels)[po][:, po]
        b2 = self.out_layers[3].bias.detach()[po].float()
        has_skip = not isinstance(self.skip_connection, nn.Identity)
        if has_skip:
            ws = self.skip_connection.weight.detach().reshape(self.out_channels, self.channels)[po][:, pi]
            w2 = torch.cat([w2, ws], dim=1)
            b2 = b2 + self.skip_connection.bias.detach()[po].float()
        # GroupNorm parameters are per flattened channel (c*sdim + s): gathered into NHWC order -> [sdim, C] tables; the kernel
        # takes per-channel gamma / beta, so position-dependent parameters are applied as sdim separate channel vectors only when
        # they differ across s (synthetic weights do; a trained checkpoint does too)
        g1 = self.in_layers[0].weight.detach()[pi].float().view(sdim, Cin)
        be1 = self.in_layers[0].bias.detach()[pi].float().view(sdim, Cin)
        g2 = self.out_layers[0].weight.detach()[po].float().view(sdim, Cout)
        be2 = self.out_layers[0].bias.detach()[po].float().view(sdim, Cout)
        return {"w1": bf16(w1), "b1": self.in_layers[2].bias.detach()[po].float().contiguous(),
                "we": bf16(self.emb_layers[1].weight.detach()[po]), "be": self.emb_layers[1].bias.detach()[po].float().contiguous(),
                "w2": bf16(w2), "b2": b2.contiguous(), "has_skip": has_skip, "sdim": sdim,
                "g1": g1.contiguous(), "be1": be1.contiguous(), "g2": g2.contiguous(), "be2": be2.contiguous()}

    _unit = {}

    @classmethod
    def _unit_affine(cls, C, device):
        """persistent (1, 0) GroupNorm parameters per channel count (no allocation / fill inside a captured step)"""
        key = (C, str(device))
        if key not in cls._unit:
            cls._unit[key] = (torch.ones(C, dtype=torch.float32, device=device), torch.zeros(C, dtype=torch.float32, device=device))
        return cls._unit[key]

    @classmethod
    def _gn_silu(cls, x, gamma, beta, eps, x2=None):
        """GroupNorm32 + SiLU over the flattened channels of [B, sdim, 1, C] (+ concat): statistics per (image, channel group) over
        all sdim positions == the reference's groups of the flattened index; gamma / beta differ per position, so the affine
        part is applied with identity parameters by the kernel's statistics pass and finished per position."""
        ops = _ops()
        B, sdim, _, C1 = x.shape
        C = C1 + (x2.shape[-1] if x2 is not None else 0)
        ones, zeros = cls._unit_affine(C, x.device)
        xn = ops.groupnorm(x, ones, zeros, eps, act=ops.ACT_NONE, x2=x2)            # (x - mean) * rstd, bf16 [B, sdim, 1, C]
        return ops.affine_silu_rows(xn.view(B, sdim * C), gamma.view(-1), beta.view(-1))

    def forward(self, x, emb):
        """x: NHWC bf16 [B, sdim, 1, C] or a pair (h, skip) == cat along C.  emb: fp32 [B, emb_channels] (SiLU applied here)."""
        ops = _ops()
        p = self.packed()
        x1, x2 = x if isinstance(x, tuple) else (x, None)
        require_cuda(x1, "FCBlock_MultiDim")
        B, sdim = x1.shape[0], x1.shape[1]
        eps = self.in_layers[0].eps
        a1 = self._gn_silu(x1, p["g1"], p["be1"], eps, x2=x2)                      # [B, sdim*Cin] bf16
        if isinstance(emb, EmbTable):
            e, bstride = emb.slot(self.emb_slot[0]), emb.total
        else:
            e = ops.linear_small(emb.float().contiguous(), p["we"], (p["be"] + p["b1"]).contiguous(), act_in=ops.ACT_SILU)
            bstride = self.out_channels
        h = ops.gemm(a1, p["w1"], bias=e, bias_bstride=bstride, rows_per_batch=1)
        Cout = self.out_channels_multidim[0]
        a2 = self._gn_silu(h.view(B, sdim, 1, Cout), p["g2"], p["be2"], self.out_layers[0].eps)
        raw = x1 if x2 is None else torch.cat([x1, x2], dim=-1)                     # (data movement only: 4 positions per row)
        raw = raw.reshape(B, -1)
        if p["has_skip"]:
            out = ops.gemm(a2, p["w2"], bias=p["b2"], a2=raw)
        else:
            out = ops.gemm(a2, p["w2"], bias=p["b2"], resid=raw)
        return out.view(B, sdim, 1, Cout)


class OutHead0D(PackedModule):
    """GroupNorm32(C) -> SiLU -> Linear_MultiDim([C, sdim, 1] -> [output_channels]) (reference openaimodel.py:2957-2962),
    registered under the reference's Sequential indices 0 (norm) and 2 (linear)."""

    def __init__(self, current_channel, output_channels):
        super().__init__()
        self.add_module("0", normalization(current_channel[0]))
        self.add_module("1", nn.SiLU())
        self.add_module("2", zero_module(Linear_MultiDim(current_channel, [output_channels], bias=True)))

    def _pack(self):
        norm = getattr(self, "0")
        return {"g": f32(norm.weight), "b": f32(norm.bias)}

    def forward(self, x):
        ops = _ops()
        p = self.packed()
        a = ops.groupnorm(x, p["g"], p["b"], getattr(self, "0").eps, act=ops.ACT_SILU)
        return getattr(self, "2")(a)


@register('openai_unet_0d_next')
class UNetModel0D_Next(UNetModel2D_Next):
    """The 0-D (text-latent) diffuser (reference openaimodel.py:2814-2975).  Image sampling only needs its context blocks (the
    text-context SpatialTransformers, vd.py:345; configs/model/openai_unet.yaml:78-81) — that is what 'vd_four_flow_v1-0' builds
    by default here.  With 'data' in parts (round 2, SURVEY §8f rank 4) the data blocks of the text-latent flows are built too:
    Linear_MultiDim / FCBlock_MultiDim on a [B, 768] latent expanded to [C, second_dim, 1] features (NHWC bf16 [B, sdim, 1, C] here)."""

    def __init__(self, input_channels, model_channels, output_channels, context_dim=788,
                 num_noattn_blocks=(2, 2, 2, 2), channel_mult=(1, 2, 4, 8), second_dim=(4, 4, 4, 4),
                 with_attn=[True, True, True, False], num_heads=8, num_head_channels=None, use_checkpoint=False,
                 parts=['global', 'data', 'context']):
        nn.Module.__init__(self)
        self.parts = parts if isinstance(parts, list) else [parts]
        self.input_channels = input_channels
        self.model_channels = model_channels
        self.output_channels = output_channels
        self.num_noattn_blocks = num_noattn_blocks
        self.channel_mult = channel_mult
        self.second_dim = second_dim
        self.with_attn = with_attn
        self.num_heads = num_heads
        self.num_head_channels = num_head_channels
        self.glayer_included = 'global' in self.parts
        self.dlayer_included = 'data' in self.parts
        self.clayer_included = 'context' in self.parts
        if len(set(second_dim)) != 1:
            raise NotImplementedError("UNetModel0D_Next: one second_dim for all levels (as in every VD config)")
        self.layer_sequence_ordering = []
        time_embed_dim = model_channels * 4
        if self.glayer_included:
            self.time_embed = nn.Sequential(linear(model_channels, time_embed_dim), nn.SiLU(), linear(time_embed_dim, time_embed_dim))
        if self.dlayer_included:
            self.data_blocks = nn.ModuleList([])
            FCBlockDefault = partial(FCBlock_MultiDim, dropout=0, use_checkpoint=use_checkpoint)
            Lin = lambda i, o: Linear_MultiDim(i, o, bias=True)
        else:
            FCBlockDefault = lambda *a, **k: None
            Lin = lambda i, o: None
        if self.clayer_included:
            self.context_blocks = nn.ModuleList([])
        CrossAttnDefault = partial(SpatialTransformer, context_dim=context_dim, disable_self_attn=False) if self.clayer_included \
            else (lambda *a, **k: None)

        def ctx(ch):
            d_head, n_heads = self.get_d_head_n_heads(ch)
            self.add_context_layer(CrossAttnDefault(in_channels=ch, d_head=d_head, n_heads=n_heads))

        sdim = second_dim[0]
        cur = [model_channels, sdim, 1]
        self.add_data_layer(Lin([input_channels], cur))
        self.layer_sequence_ordering.append('save_hidden_feature')
        input_block_channels = [cur]
        for level_idx, (mult, sdim) in enumerate(zip(channel_mult, second_dim)):
            for _ in range(num_noattn_blocks[level_idx]):
                self.add_data_layer(FCBlockDefault(cur, time_embed_dim, out_channels=[mult * model_channels, sdim, 1]))
                cur = [mult * model_channels, sdim, 1]
                if with_attn[level_idx]:
                    ctx(cur[0])
                input_block_channels.append(cur)
                self.layer_sequence_ordering.append('save_hidden_feature')
            if level_idx != len(channel_mult) - 1:
                self.add_data_layer(Lin(cur, cur))
                input_block_channels.append(cur)
                self.layer_sequence_ordering.append('save_hidden_feature')
        self.i_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_sequence_ordering = []
        self.add_data_layer(FCBlockDefault(cur, time_embed_dim))
        ctx(cur[0])
        self.add_data_layer(FCBlockDefault(cur, time_embed_dim))
        self.m_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_sequence_ordering = []
        for level_idx, (mult, sdim) in list(enumerate(zip(channel_mult, second_dim)))[::-1]:
            for _ in range(num_noattn_blocks[level_idx] + 1):
                self.layer_sequence_ordering.append('load_hidden_feature')
                extra = input_block_channels.pop()
                self.add_data_layer(FCBlockDefault([cur[0] + extra[0]] + cur[1:], time_embed_dim,
                                                   out_channels=[mult * model_channels, sdim, 1]))
                cur = [mult * model_channels, sdim, 1]
                if with_attn[level_idx]:
                    ctx(cur[0])
            if level_idx != 0:
                self.add_data_layer(Lin(cur, cur))
        self.add_data_layer(OutHead0D(cur, output_channels) if self.dlayer_included else None)
        self.o_order = copy.deepcopy(self.layer_sequence_ordering)
        self.layer_order = copy.deepcopy(self.i_order + self.m_order + self.o_order)
        del self.layer_sequence_ordering
        self.parameter_group = {}
        if self.glayer_included:
            self.parameter_group['global'] = self.time_embed
        if self.dlayer_included:
            self.parameter_group['data'] = self.data_blocks
        if self.clayer_included:
            self.parameter_group['context'] = self.context_blocks
        self._emb_packed = None
        self._assign_emb_slots()

    def _fc_blocks(self):
        return [layer for blk in self.data_blocks for layer in blk if isinstance(layer, FCBlock_MultiDim)] if self.dlayer_included else []

    def _assign_emb_slots(self):
        off = 0
        for layer in self._fc_blocks():
            layer.emb_slot = (off, None)
            off += layer.out_channels
        self._emb_total = off

    def _pack_emb(self):
        if self._emb_packed is None:
            with torch.no_grad():
                ps = [layer.packed() for layer in self._fc_blocks()]
                self._emb_packed = {"w": torch.cat([q["we"] for q in ps], 0).contiguous(),
                                    "b": torch.cat([q["be"] + q["b1"] for q in ps], 0).contiguous()}
        return self._emb_packed

    def embed_table(self, t_emb, time_owner=None):
        """Sinusoid [B, model_channels] fp32 -> EmbTable: the time_embed MLP, then the SiLU -> Linear of EVERY FCBlock as one
        [B, sum(C*sdim)] tensor-core GEMM with the first conv's bias folded in (columns in each block's NHWC order).  Per block
        and step this was otherwise a CUDA-core launch of its own.
        Without data blocks (context-only build) the raw embedding is returned."""
        if not self.dlayer_included:
            return (time_owner or self).time_embedding(t_emb)
        ops = _ops()
        w0, b0, w2, b2 = (time_owner or self).time_embed_packed()
        p = self._pack_emb()
        h = ops.gemm(ops.to_bf16(t_emb.contiguous()), w0, bias=b0, act=ops.ACT_SILU, ksplit=1)
        s = ops.gemm(h, w2, bias=b2, act=ops.ACT_SILU, ksplit=1)          # SiLU(time_embed(t_emb)), bf16
        return EmbTable(ops.gemm(s, p["w"], bias=p["b"], out_dtype=torch.float32, ksplit=1))

    def forward(self, *a, **k):
        raise NotImplementedError("the 0-D diffuser is driven by VD_v2_0.apply_model (data blocks of diffuser[x_type], context blocks of diffuser[c_type])")
