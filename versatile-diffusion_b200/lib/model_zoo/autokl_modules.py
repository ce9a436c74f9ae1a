"""kl-f8 Encoder / Decoder of AutoencoderKL on vdb200 kernels
(reference lib/model_zoo/autokl_modules.py:38-141 blocks, :150-202 AttnBlock, :368-459 Encoder, :462-568 Decoder).
Same constructor keywords and parameter names (down.{l}.block.{b}.{norm1,conv1,norm2,conv2,nin_shortcut},
mid.{block_1,attn_1,block_2}, up.{l}.upsample.conv, norm_out, conv_out).  NHWC bf16 inside; GN eps 1e-6.
"""
import numpy as np
import torch
import torch.nn as nn

from .diffusion_utils import (PackedMixin, PackedModule, bf16, f32, pack_conv1x1, pack_conv3x3, require_cuda,
                              fold_upsample_conv3x3, upsample_fold_enabled)


def _ops():
    from vdb200 import ops
    return ops


def Normalize(in_channels, num_groups=32):
    return torch.nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


class Upsample(PackedModule):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        if not self.with_conv:
            return {}
        d = {"w": pack_conv3x3(self.conv.weight), "b": f32(self.conv.bias)}
        if upsample_fold_enabled(1 << 30, self.conv.out_channels):   # (the folded copy is only built when some input can use it)
            d["wf"] = fold_upsample_conv3x3(self.conv.weight)
        return d

    def forward(self, x):
        ops = _ops()
        if self.with_conv and upsample_fold_enabled(x.shape[0] * x.shape[1] * x.shape[2], self.conv.out_channels):
            p = self.packed()
            return ops.upsample2x_conv3x3_folded(x, p["wf"], bias=p["b"])     # 2.25x fewer FLOPs, no upsampled temporary
        x = ops.upsample2x(x)
        if self.with_conv:
            p = self.packed()
            x = ops.conv3x3(x, p["w"], bias=p["b"])
        return x


class Downsample(PackedModule):
    """pad (0,1,0,1) + 3x3 stride-2 conv (reference :60-79) == conv mode 2 of the implicit-GEMM kernel."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        if not with_conv:
            raise NotImplementedError("avg-pool downsample is not used by kl-f8")
        self.with_conv = with_conv
        self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def _pack(self):
        return {"w": pack_conv3x3(self.conv.weight), "b": f32(self.conv.bias)}

    def forward(self, x):
        p = self.packed()
        return _ops().conv3x3(x, p["w"], bias=p["b"], mode=2)


class ResnetBlock(PackedModule):
    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        if conv_shortcut or temb_channels > 0:
            raise NotImplementedError("kl-f8 uses nin_shortcut and no timestep embedding")
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = Normalize(out_channels)
        self.dropout = torch.nn.Dropout(dropout)
        self.conv2 = torch.nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def _pack(self):
        w2, b2 = pack_conv3x3(self.conv2.weight), f32(self.conv2.bias)
        has_skip = self.in_channels != self.out_channels
        if has_skip:
            w2 = torch.cat([w2, pack_conv1x1(self.nin_shortcut.weight)], 1).contiguous()
            b2 = (b2 + f32(self.nin_shortcut.bias)).contiguous()
        return {"g1": f32(self.norm1.weight), "be1": f32(self.norm1.bias), "w1": pack_conv3x3(self.conv1.weight),
                "b1": f32(self.conv1.bias), "g2": f32(self.norm2.weight), "be2": f32(self.norm2.bias),
                "w2": w2, "b2": b2, "has_skip": has_skip}

    def forward(self, x, temb=None):
        ops = _ops()
        p = self.packed()
        a1 = ops.groupnorm(x, p["g1"], p["be1"], self.norm1.eps, act=ops.ACT_SILU)
        h = ops.conv3x3(a1, p["w1"], bias=p["b1"])
        a2 = ops.groupnorm(h, p["g2"], p["be2"], self.norm2.eps, act=ops.ACT_SILU)
        if p["has_skip"]:
            return ops.conv3x3(a2, p["w2"], bias=p["b2"], skip1=x)
        return ops.conv3x3(a2, p["w2"], bias=p["b2"], resid=x)


class AttnBlock(PackedModule):
    """Single-head spatial self-attention with d = C = 512 (reference :150-202).  d exceeds the flash attention
    kernel's d_head limit (160), and it runs once per decode, so it is three wgmma GEMMs around a row softmax:
    S = q k^T (bf16), P = softmax(S * C^-1/2) (bf16), O = P v (+ b_v: rows of P sum to 1), proj_out + x."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)

    def _pack(self):
        wqk = torch.cat([pack_conv1x1(self.q.weight), pack_conv1x1(self.k.weight)], 0).contiguous()
        bqk = torch.cat([f32(self.q.bias), f32(self.k.bias)], 0).contiguous()
        return {"g": f32(self.norm.weight), "b": f32(self.norm.bias), "wqk": wqk, "bqk": bqk,
                "wv": pack_conv1x1(self.v.weight), "bv": f32(self.v.bias),
                "wo": pack_conv1x1(self.proj_out.weight), "bo": f32(self.proj_out.bias)}

    def forward(self, x):
        ops = _ops()
        p = self.packed()
        B, H, W, C = x.shape
        N = H * W
        hn = ops.groupnorm(x, p["g"], p["b"], self.norm.eps).view(B * N, C)
        qk = ops.gemm(hn, p["wqk"], bias=p["bqk"])                 # [B*N, 2C]
        o = torch.empty(B * N, C, dtype=torch.bfloat16, device=x.device)
        for b in range(B):
            rows = slice(b * N, (b + 1) * N)
            s = ops.gemm(qk[rows, :C], qk[rows, C:])               # [N, N] = q k^T
            pm = ops.softmax_rows(s, scale=float(int(C) ** (-0.5)))
            vt = ops.gemm(p["wv"], hn[rows])                       # [C, N] = (W_v h^T), bias folded below
            ops.gemm(pm, vt, bias=p["bv"], out=o[rows])
        out = ops.gemm(o, p["wo"], bias=p["bo"], resid=x.view(B * N, C))
        return out.view(B, H, W, C)


def make_attn(in_channels, attn_type="vanilla"):
    assert attn_type in ["vanilla", "none"], f'attn_type {attn_type} is not on the kl-f8 path'
    print(f"making attention of type '{attn_type}' with {in_channels} in_channels")
    return AttnBlock(in_channels) if attn_type == "vanilla" else nn.Identity()


class ConvSmallIn(PackedMixin, nn.Conv2d):
    """3x3 conv whose input has < 8 channels (latent z: 4, RGB: 3): fp32 NHWC -> im2col (K -> 64) -> GEMM."""

    def __init__(self, in_channels, out_channels):
        super().__init__(in_channels, out_channels, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        w = self.weight.detach()
        n, cin = w.shape[0], w.shape[1]
        wp = torch.zeros(n, 64, dtype=torch.bfloat16, device=w.device)
        wp[:, :9 * cin] = w.permute(0, 2, 3, 1).reshape(n, -1).to(torch.bfloat16)
        return {"w": wp, "b": f32(self.bias)}

    def forward(self, x, in_scale=1.0, in_shift=0.0):
        ops = _ops()
        p = self.packed()
        B, H, W, _ = x.shape
        col = ops.im2col3x3_small(x, kpad=64, in_scale=in_scale, in_shift=in_shift)
        return ops.gemm(col, p["w"], bias=p["b"]).view(B, H, W, -1)


class _Level(nn.Module):
    pass


class Encoder(PackedModule):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        if use_linear_attn or len(attn_resolutions):
            raise NotImplementedError("kl-f8 has attention only in the mid block")
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.conv_in = ConvSmallIn(in_channels, self.ch)
        in_ch_mult = (1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
        self.down = nn.ModuleList()
        block_in = ch
        for i_level in range(self.num_resolutions):
            block = nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
            down = _Level()
            down.block = block
            down.attn = nn.ModuleList()
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
            self.down.append(down)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        return {"g": f32(self.norm_out.weight), "b": f32(self.norm_out.bias), "w": pack_conv3x3(self.conv_out.weight),
                "bc": f32(self.conv_out.bias)}

    def forward(self, x, in_scale=1.0, in_shift=0.0):
        """x: fp32 NHWC [B,H,W,3] -> fp32 NHWC moments-before-quant [B,H/8,W/8,2*z] (reference :434-459)."""
        ops = _ops()
        h = self.conv_in(x, in_scale, in_shift)
        for i_level in range(self.num_resolutions):
            for i_block in range(self.num_res_blocks):
                h = self.down[i_level].block[i_block](h)
            if i_level != self.num_resolutions - 1:
                h = self.down[i_level].downsample(h)
        h = self.mid.block_1(h)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h)
        p = self.packed()
        a = ops.groupnorm(h, p["g"], p["b"], self.norm_out.eps, act=ops.ACT_SILU)
        return ops.conv3x3(a, p["w"], bias=p["bc"], out_dtype=torch.float32)


class Decoder(PackedModule):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if use_linear_attn or len(attn_resolutions) or give_pre_end or tanh_out:
            raise NotImplementedError("only the kl-f8 decoder configuration is built")
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.give_pre_end = give_pre_end
        self.tanh_out = tanh_out
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        print("Working with z of shape {} = {} dimensions.".format(self.z_shape, np.prod(self.z_shape)))
        self.conv_in = ConvSmallIn(z_channels, block_in)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
            up = _Level()
            up.block = block
            up.attn = nn.ModuleList()
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        return {"g": f32(self.norm_out.weight), "b": f32(self.norm_out.bias), "w": pack_conv3x3(self.conv_out.weight),
                "bc": f32(self.conv_out.bias)}

    def forward(self, z):
        """z: fp32 NHWC [B,h,w,z_channels] (after post_quant_conv) -> fp32 NHWC [B,8h,8w,out_ch] (reference :535-568)."""
        ops = _ops()
        self.last_z_shape = z.shape
        h = self.conv_in(z)
        h = self.mid.block_1(h)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h)
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                h = self.up[i_level].block[i_block](h)
            if i_level != 0:
                h = self.up[i_level].upsample(h)
        p = self.packed()
        a = ops.groupnorm(h, p["g"], p["b"], self.norm_out.eps, act=ops.ACT_SILU)
        return ops.conv3x3(a, p["w"], bias=p["bc"], out_dtype=torch.float32)
