"""Every UNet, text-diffuser and VAE layer module (openaimodel.py, attention.py, autokl_modules.py) on its own against fp64, at
every configuration the full-size models build.

The kernels have their own per-element tests.  What this file checks is the layer code that wires them: the folded LayerNorm
(bf16(W gamma) and its column sums), head padding, the context padded to Lp = ceil(L / 8) 8 rows of which only L are keys, the
ragged self-attention copy, the GEGLU row order, the ResBlock emb slots and its skip conv as extra K columns with the bias folded
into b2, the mixing ratio / accumulator of proj_out, the 0-D diffuser's row / column permutations and per-position GroupNorm
tables, and the VAE AttnBlock's three GEMMs around softmax_rows with b_v added after P v.

References.  Each case runs one module of the product on a bf16 input and builds two fp64 references on the CPU from the same
parameters and the same bf16 input, both through the oracle's own function for that layer (oracle/vd_oracle.py, pinned to the
unmodified reference by test_oracle):
  ref   the oracle in fp64.
  twin  the same evaluation with the product's storage roundings: every weight rounded to bf16 (where a LayerNorm is folded
        into a projection, the projection reads bf16(W gamma) / gamma, from the identity of include/vdb200.h: W' = W0 gamma
        rounded to bf16), and every activation the product stores in bf16 rounded to bf16 through the oracle's rounding hook
        (GroupNorm / SiLU outputs, conv1, tokens after proj_in and after each residual, LayerNorm outputs where they are not
        folded, q / k / v, the attention output, the GEGLU hidden, S and P of the VAE attention, the module output).  Flash
        attention rounds its unnormalised weights to bf16 for P V only; the twin does the same with exp(s - max).
  The twin restates where the product rounds, never how it packs: permutations, head padding, the GEGLU order, emb slots
  and fused skip columns are not in it, so a packing defect cannot be copied into both sides.

Pass criterion, per slice (one batch item x one 32-channel group x up to 4096 positions, so a defect confined to one head,
tile, item or emb slot shows in its own slice), u = 2^-24:
    rms(out - ref) <= RHO rms(twin - ref) + u rms(ref)        max|out - ref| <= RHO_MAX max|twin - ref| + u max|ref|
and, against the twin itself,
    rms(out - twin) <= KAPPA rms(twin - ref) + u rms(ref)
The product and the twin round at the same points, so the ratio sits near 1.  What the twin does not restate, and why it
stays within the ratios:
  - fp32 accumulation and its order (GEMM tiles, split-K, the GroupNorm / LayerNorm sums): ~2^-24 sqrt(K) relative, far
    below one bf16 rounding.
  - the folded LayerNorm's mean / rstd come from the fp32 sums of the producing GEMM before its bf16 rounding, while the
    twin normalises the rounded tokens; the two statistics differ by the mean of C rounding errors, 2^-9 / sqrt(C) of the
    token magnitude, below the rounding of the tokens themselves.
  - flash attention's running maximum (rescaled lazily, up to 2^8 above the final one) shifts where bf16(P) rounds; the
    rounding has the same relative size, not the same values.
  - the folded Upsample rounds the sums of up to four 3x3 taps to bf16 (fold_upsample_conv3x3), the twin each tap: the same
    relative rounding of the weights, on different values.
  - ex2 / tanh.approx in the kernels' exp and SiLU: 2^-22 and 2^-11 relative, below the bf16 rounding of their outputs.

The out - twin bound is what sees a defect of the same size as a rounding both sides share.  The folded LayerNorm's column
sums are one: summed over the unrounded W gamma they add r mu (sum W gamma - sum bf16(W gamma)) to each projection, about
2^-9 mu / sigma, the size of the tokens' own bf16 rounding; that rounding is in both out and twin, so out - ref grows only by
a factor near sqrt(2) and RHO cannot see it, while out - twin doubles.  Where the token rows have mean / std 64 and the
LayerNorm is folded, the tokens' rounding (identical in product and twin) is most of twin - ref, and out - twin, which does
not contain it, stays below 0.7 of it (0.59 - 0.68 measured): those rows take KAPPA_SHARED = 0.85.  Elsewhere out - twin is
the product's own arithmetic (the GroupNorm's E[x^2] - mean^2 in fp32, tanh.approx in SiLU, flash attention's lazy maximum,
the folded Upsample's weights) against the twin's: up to 1.50 of twin - ref (folded Upsample), 1.24 (four-token
SpatialTransformer), <= 0.9 in every other class; KAPPA = 1.6.

RHO and RHO_MAX were set from the H100 runs (H100 80GB HBM3, 700 W limit).  Worst slice ratios per module class, rms / max:
Upsample 1.23 / 1.51 (folded), SpatialTransformer 1.20 / 1.63 (the four-token 0-D ones), VAE Upsample 1.12 / 1.36 (folded),
the every-slot rows 1.11 / 1.37, FCBlock 1.06 / 1.14, OutHead0D 1.03 / 1.07, ResBlock 1.02 / 1.12, and at most 1.01 / 1.06
for OutHead, VAE ResnetBlock, AttnBlock, Downsample, ConvIn, Linear_MultiDim and the time MLP.

Inputs: GroupNorm groups and LayerNorm token rows with mean / std of 0, 8 and 64 (token means through proj_in's bias), one
constant group, VAE inputs with |x| up to ~1e3, contexts of 77 and 257 tokens that share a component across tokens, biases at
unit scale (BIAS_SCALE).

Cases.  CASES holds one row per module configuration of the full-size 2-D UNet (B 2 at the 64x64 latent, B 8 at its 16x16
and 8x8 levels, B 3 at a 40x56 latent whose 10x14 and 5x7 levels have H W % 8 != 0), the 0-D text diffuser (four tokens) and
the kl-f8 VAE at 512^2 (B 1), plus the stand-alone and embed_all emb sources, a dual-context mixing row (0.7, 0.3), a plain VAE
Upsample and the mini UNet's d_head 8 / 16 / 32 transformers.  The slot rows then run every ResBlock of the 2-D UNet and every
FCBlock of the 0-D diffuser once at a small size, so each reads its own slot of the owner's EmbTable.
test_every_configuration_has_a_case walks the full-size models and fails on a configuration without a row;
test_every_path_reached checks that the branches and every slot were taken, through the predicates the code branches on.
The configuration walk and the identity-hook check build their modules on the meta device or the CPU and need no GPU.
"""
import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
U = 2.0 ** -24
RHO, RHO_MAX = 1.5, 2.5
KAPPA, KAPPA_SHARED = 1.6, 0.85
BIAS_SCALE = 50.0          # synthetic biases are 0.02 randn: at unit scale a bias dropped or added twice shows
SEED = 1
SLICE_POS, SLICE_CH = 4096, 32
REACHED = set()
RAN = set()


def O():
    from oracle import vd_oracle
    return vd_oracle


def bf(t):
    return t.to(torch.bfloat16).to(torch.float64)


def rounding(*names):
    names = set(names)
    return lambda name, t: bf(t) if name in names else t


def identity(name, t):
    return t


# ---------------------------------------------------------------------------------------------------------------------------
# the models the configurations come from
# ---------------------------------------------------------------------------------------------------------------------------
UNET2D = dict(in_channels=4, out_channels=4, model_channels=320, attention_resolutions=[4, 2, 1], num_res_blocks=[2, 2, 2, 2],
              channel_mult=[1, 2, 4, 4], num_heads=8, context_dim=768)
UNET0D = dict(input_channels=768, model_channels=320, output_channels=768, num_noattn_blocks=[2, 2, 2, 2], channel_mult=[1, 2, 4, 4],
              second_dim=[4, 4, 4, 4], with_attn=[True, True, True, False], num_heads=8, context_dim=768)
VAE = dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
           attn_resolutions=[], dropout=0.0)
DRIVES_2D = [(2, 64, 64, None), (8, 64, 64, {16, 8}), (3, 40, 56, None)]     # (B, H, W, latent sides walked: None = all)
CONTEXTS = (77, 257)
VAE_IMAGE = 512


def build(cls, kw, device, fill=True):
    """the module on `device` with the synthetic weights of oracle/weights.py (construction on meta: no init cost)"""
    from oracle import weights
    with torch.device("meta"):
        m = cls(**kw)
    if device == "meta":
        return m
    m = m.to_empty(device=device)
    if fill:
        fill_weights(m, "")
    return m.eval()


def fill_weights(m, key):
    from oracle import weights
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(weights.tensor_for(key + k, p.shape, SEED) * (BIAS_SCALE if k.endswith("bias") else 1.0))


def _unet_classes():
    from lib.model_zoo import openaimodel as om
    return om


def walk_2d(net, B, H, W, levels=None):
    """(module, B, H, W, pair) of every data / context block in execution order (the walk of openaimodel.unet_walk); pair is
    (channels of h, channels of the skip) for a block whose input is the pair (h, skip), else None.  levels: the latent sides
    walked (None: all)"""
    om = _unet_classes()
    out, hs, h, w, ch, pair = [], [], H, W, None, None
    d_it, c_it = iter(net.data_blocks), iter(net.context_blocks) if net.clayer_included else None
    for kind in net.i_order + net.m_order + net.o_order:
        if kind == "d":
            m = next(d_it)[0]
            if levels is None or h in levels:
                out.append((m, B, h, w, pair))
            pair = None
            if isinstance(m, om.Downsample):
                h, w = (h + 1) // 2, (w + 1) // 2
            elif isinstance(m, om.Upsample):
                h, w = 2 * h, 2 * w
            elif isinstance(m, (om.ConvIn, om.ResBlock)):
                ch = m.out_channels
        elif kind == "c" and c_it is not None:
            m = next(c_it)[0]
            if levels is None or h in levels:
                out.append((m, B, h, w, None))
        elif kind == "save_hidden_feature":
            hs.append(ch)
        elif kind == "load_hidden_feature":
            pair = (ch, hs.pop())
    return out


def walk_0d(net, B=2):
    """the same for the 0-D diffuser: four tokens, NHWC [B, 4, 1, C]"""
    om = _unet_classes()
    out, hs, ch, pair = [], [], None, None
    d_it, c_it = iter(net.data_blocks), iter(net.context_blocks) if net.clayer_included else None
    for kind in net.i_order + net.m_order + net.o_order:
        if kind == "d":
            m = next(d_it)[0]
            out.append((m, B, 4, 1, pair))
            pair = None
            if isinstance(m, om.Linear_MultiDim):
                ch = m.out_features_multidim[0]
            elif isinstance(m, om.FCBlock_MultiDim):
                ch = m.out_channels_multidim[0]
        elif kind == "c" and c_it is not None:
            out.append((next(c_it)[0], B, 4, 1, None))
        elif kind == "save_hidden_feature":
            hs.append(ch)
        elif kind == "load_hidden_feature":
            pair = (ch, hs.pop())
    return out


def walk_vae(enc, dec, size=VAE_IMAGE):
    out, h = [], size
    for lvl in range(enc.num_resolutions):
        for blk in enc.down[lvl].block:
            out.append((blk, 1, h, h, False))
        if lvl != enc.num_resolutions - 1:
            out.append((enc.down[lvl].downsample, 1, h, h, False))
            h //= 2
    mids = lambda m, h: [(m.mid.block_1, 1, h, h, False), (m.mid.attn_1, 1, h, h, False), (m.mid.block_2, 1, h, h, False)]
    out += mids(enc, h)
    out += mids(dec, h)
    for lvl in reversed(range(dec.num_resolutions)):
        for blk in dec.up[lvl].block:
            out.append((blk, 1, h, h, False))
        if lvl != 0:
            out.append((dec.up[lvl].upsample, 1, h, h, False))
            h *= 2
    return out


def signatures(m, B, H, W, pair):
    """the configuration signature(s) of one module at one input shape; a SpatialTransformer has one per context length"""
    om = _unet_classes()
    from lib.model_zoo import attention as at
    from lib.model_zoo import autokl_modules as ak
    from lib.model_zoo.diffusion_utils import upsample_fold_enabled
    if isinstance(m, om.ResBlock):
        skip = "pair" if pair else ("conv" if not isinstance(m.skip_connection, torch.nn.Identity) else "identity")
        return [("ResBlock", m.channels, m.out_channels, H, W, skip, "table")]
    if isinstance(m, at.SpatialTransformer):
        blk = m.transformer_blocks[0]
        inner = blk.attn1.heads * blk.attn1.dim_head
        fold = at.ln_fold_fits(inner, B, H, W)
        return [("SpatialTransformer", m.in_channels, blk.attn1.heads, blk.attn1.dim_head, H, W, L,
                 "fold" if fold else "plain", "ragged" if (H * W) % 8 else "aligned", "single") for L in CONTEXTS]
    if isinstance(m, om.ConvIn):
        return [("ConvIn", m.in_channels, m.out_channels, H, W)]
    if isinstance(m, om.Downsample):
        return [("Downsample", m.channels, H, W)]
    if isinstance(m, om.Upsample):
        return [("Upsample", m.channels, H, W, "fold" if upsample_fold_enabled(B * H * W, m.out_channels) else "plain")]
    if isinstance(m, om.OutHead):
        return [("OutHead", getattr(m, "0").num_channels, getattr(m, "2").out_channels, H, W)]
    if isinstance(m, om.FCBlock_MultiDim):
        skip = "pair" if pair else ("conv" if not isinstance(m.skip_connection, torch.nn.Identity) else "identity")
        return [("FCBlock_MultiDim", m.channels_multidim[0], m.out_channels_multidim[0], H, skip, "table")]
    if isinstance(m, om.Linear_MultiDim):
        return [("Linear_MultiDim", tuple(m.in_features_multidim), tuple(m.out_features_multidim))]
    if isinstance(m, om.OutHead0D):
        return [("OutHead0D", getattr(m, "0").num_channels, getattr(m, "2").out_features)]
    if isinstance(m, ak.ResnetBlock):
        return [("vae.ResnetBlock", m.in_channels, m.out_channels, H, W)]
    if isinstance(m, ak.AttnBlock):
        return [("vae.AttnBlock", m.in_channels, H, W)]
    if isinstance(m, ak.Upsample):
        return [("vae.Upsample", m.conv.in_channels, H, W, "fold" if upsample_fold_enabled(B * H * W, m.conv.out_channels) else "plain")]
    if isinstance(m, ak.Downsample):
        return [("vae.Downsample", m.conv.in_channels, H, W)]
    raise AssertionError(f"no signature for {type(m).__name__}")


# ---------------------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------------------
def res(cin, cout, skip, B, H, W, emb="table", nth=0):
    return dict(kind="res", cin=cin, cout=cout, skip=skip, B=B, H=H, W=W, emb=emb, nth=nth,
                id=f"res-{cin}-{cout}-{skip}-{emb}-b{B}-{H}x{W}")


def st(C, B, H, W, L, tok_mean=0.0, heads=8, mix=None):
    from lib.model_zoo.attention import ln_fold_fits
    kappa = KAPPA_SHARED if tok_mean >= 64 and ln_fold_fits(C, B, H, W) else KAPPA
    return dict(kind="st", C=C, heads=heads, B=B, H=H, W=W, L=L, tok_mean=tok_mean, mix=mix, kappa=kappa,
                id=f"st-{C}-h{heads}-b{B}-{H}x{W}-L{L}" + ("-mix" if mix else "") + (f"-mean{int(tok_mean)}" if tok_mean else ""))


def conv(cls, C, B, H, W, cout=None):
    return dict(kind=cls, C=C, cout=cout, B=B, H=H, W=W, id=f"{cls}-{C}-b{B}-{H}x{W}")


def fc(cin, cout, skip, emb="table", B=3):
    return dict(kind="fc", cin=cin, cout=cout, skip=skip, emb=emb, B=B, id=f"fc-{cin}-{cout}-{skip}-{emb}")


def lin(fin, fout, B=3):
    return dict(kind="lin", fin=fin, fout=fout, B=B, id=f"lin-{'x'.join(map(str, fin))}-{'x'.join(map(str, fout))}")


def vres(cin, cout, H, B=1):
    return dict(kind="vres", cin=cin, cout=cout, B=B, H=H, W=H, id=f"vres-{cin}-{cout}-{H}")


RES_LEVELS = [  # (cin, cout, skip, level divisor)
    (320, 320, "identity", 1), (320, 640, "conv", 2), (640, 640, "identity", 2), (640, 1280, "conv", 4), (1280, 1280, "identity", 4),
    (1280, 1280, "identity", 8), (2560, 1280, "pair", 8), (2560, 1280, "pair", 4), (1920, 1280, "pair", 4), (1920, 640, "pair", 2),
    (1280, 640, "pair", 2), (960, 640, "pair", 2), (960, 320, "pair", 1), (640, 320, "pair", 1)]
ST_LEVELS = [(320, 1), (640, 2), (1280, 4), (1280, 8)]


def slot_rows():
    """every ResBlock of the 2-D UNet and every FCBlock of the 0-D diffuser once, at a small size, reading its own slot of the
    owner's EmbTable (the rows above take one block per configuration)"""
    from oracle import vd_oracle
    rows = [dict(kind="res", idx=i, B=2, H=8, W=8, emb="table", id=f"slot-res-{i}")
            for kind, i, _ in vd_oracle.unet_layout() if kind == "res"]
    return rows + [dict(kind="fc", idx=i, B=2, emb="table", id=f"slot-fc-{i}") for kind, i in vd_oracle.unet0d_layout() if kind == "fc"]

CASES = (
    [res(ci, co, sk, 2, 64 // d, 64 // d) for ci, co, sk, d in RES_LEVELS]
    + [res(ci, co, sk, 3, 40 // d, 56 // d, nth=-1) for ci, co, sk, d in RES_LEVELS]
    + [res(320, 320, "identity", 2, 16, 16, emb="emb"), res(1920, 640, "pair", 2, 8, 8, emb="all"),
       res(320, 640, "conv", 3, 8, 8, emb="all", nth=-1)]
    + [st(C, 2, 64 // d, 64 // d, L, tok_mean=(0.0, 8.0, 64.0)[(i + j) % 3]) for i, (C, d) in enumerate(ST_LEVELS)
       for j, L in enumerate(CONTEXTS)]
    + [st(C, 3, 40 // d, 56 // d, L, tok_mean=(64.0, 0.0, 8.0)[(i + j) % 3]) for i, (C, d) in enumerate(ST_LEVELS)
       for j, L in enumerate(CONTEXTS)]
    + [st(C, 3, 4, 1, L, tok_mean=8.0 * j) for C in (320, 640, 1280) for j, L in enumerate(CONTEXTS)]
    + [st(640, 2, 32, 32, 77, mix=(0.7, 0.3), tok_mean=8.0),
       st(64, 2, 16, 16, 77, tok_mean=64.0), st(128, 2, 8, 8, 77), st(256, 3, 4, 4, 257, tok_mean=8.0)]   # mini UNet: d 8 / 16 / 32
    + [conv("convin", 4, 2, 64, 64, 320), conv("convin", 4, 3, 40, 56, 320), conv("outhead", 320, 2, 64, 64, 4),
       conv("outhead", 320, 3, 40, 56, 4)]
    + [conv("down", C, 2, 64 // d, 64 // d) for C, d in ((320, 1), (640, 2), (1280, 4))]
    + [conv("down", C, 3, 40 // d, 56 // d) for C, d in ((320, 1), (640, 2), (1280, 4))]
    + [conv("up", 1280, 2, 8, 8), conv("up", 1280, 2, 16, 16), conv("up", 640, 2, 32, 32), conv("up", 1280, 8, 16, 16),
       conv("up", 1280, 3, 5, 7), conv("up", 1280, 3, 10, 14), conv("up", 640, 3, 20, 28)]
    + [dict(kind="time", B=3, id="time-embed")]
    + [lin((768,), (320, 4, 1))] + [lin((C, 4, 1), (C, 4, 1)) for C in (320, 640, 1280)]
    + [fc(320, 320, "identity"), fc(320, 640, "conv"), fc(640, 640, "identity"), fc(640, 1280, "conv"), fc(1280, 1280, "identity"),
       fc(2560, 1280, "pair"), fc(1920, 1280, "pair"), fc(1920, 640, "pair"), fc(1280, 640, "pair"), fc(960, 640, "pair"),
       fc(960, 320, "pair"), fc(640, 320, "pair"), fc(640, 1280, "conv", emb="emb", B=2)]
    + [dict(kind="out0d", C=320, B=3, id="outhead0d")]
    + [vres(512, 512, 64), vres(512, 512, 128), vres(512, 256, 256), vres(256, 256, 256), vres(256, 128, 512), vres(128, 128, 512),
       vres(128, 256, 256), vres(256, 512, 128)]
    + [dict(kind="vattn", C=512, B=1, H=64, W=64, id="vattn-512-64")]
    + [conv("vup", C, 1, H, H) for C, H in ((512, 64), (512, 128), (256, 256), (512, 32))]
    + [conv("vdown", C, 1, H, H) for C, H in ((128, 512), (256, 256), (512, 128))]
    + slot_rows()
)


def case_signature(c):
    from lib.model_zoo import attention as at
    from lib.model_zoo.diffusion_utils import upsample_fold_enabled
    k = c["kind"]
    if "idx" in c:
        return ("slot", k, c["idx"])
    if k == "res":
        return ("ResBlock", c["cin"], c["cout"], c["H"], c["W"], c["skip"], c["emb"])
    if k == "st":
        fold = at.ln_fold_fits(c["C"], c["B"], c["H"], c["W"])
        return ("SpatialTransformer", c["C"], c["heads"], c["C"] // c["heads"], c["H"], c["W"], c["L"], "fold" if fold else "plain",
                "ragged" if (c["H"] * c["W"]) % 8 else "aligned", "mix" if c["mix"] else "single")
    if k == "convin":
        return ("ConvIn", c["C"], c["cout"], c["H"], c["W"])
    if k == "down":
        return ("Downsample", c["C"], c["H"], c["W"])
    if k == "up":
        return ("Upsample", c["C"], c["H"], c["W"], "fold" if upsample_fold_enabled(c["B"] * c["H"] * c["W"], c["C"]) else "plain")
    if k == "outhead":
        return ("OutHead", c["C"], c["cout"], c["H"], c["W"])
    if k == "fc":
        return ("FCBlock_MultiDim", c["cin"], c["cout"], 4, c["skip"], c["emb"])
    if k == "lin":
        return ("Linear_MultiDim", c["fin"], c["fout"])
    if k == "out0d":
        return ("OutHead0D", c["C"], 768)
    if k == "vres":
        return ("vae.ResnetBlock", c["cin"], c["cout"], c["H"], c["W"])
    if k == "vattn":
        return ("vae.AttnBlock", c["C"], c["H"], c["W"])
    if k == "vup":
        return ("vae.Upsample", c["C"], c["H"], c["W"], "fold" if upsample_fold_enabled(c["B"] * c["H"] * c["W"], c["C"]) else "plain")
    if k == "vdown":
        return ("vae.Downsample", c["C"], c["H"], c["W"])
    return ("time",)


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
def gen(seed):
    return torch.Generator().manual_seed(seed)


def act_input(B, P, C, seed, scale=1.0):
    """[B, P, C] bf16: group g of item b has std s in [0.5, 2] scale and mean (0, 8, 64)[g % 3] s (random sign); channels of a
    group carry extra means in [-s/2, s/2]; group 3 is constant"""
    g = gen(seed)
    G = 32 if C % 32 == 0 else 1
    cpg = C // G
    sig = (torch.rand(B, G, generator=g) * 1.5 + 0.5) * scale
    ratio = torch.tensor([0.0, 8.0, 64.0]).repeat(11)[:G]
    sign = torch.where(torch.rand(B, G, generator=g) < 0.5, -1.0, 1.0)
    sig_c = sig.repeat_interleave(cpg, 1)
    mean_c = (ratio * sig * sign).repeat_interleave(cpg, 1) + (torch.rand(B, C, generator=g) - 0.5) * sig_c
    x = torch.randn(B, P, C, generator=g) * sig_c[:, None] + mean_c[:, None]
    if G == 32:
        x[:, :, 3 * cpg:4 * cpg] = 2.5 * scale
    return x.to(torch.bfloat16)


def nhwc(x, B, H, W):
    return x.view(B, H, W, -1)


def to_nchw64(x):
    return x.double().permute(0, 3, 1, 2).contiguous()


def from_nchw(y):
    """[B, C, H, W] -> [B, H W, C]"""
    return y.permute(0, 2, 3, 1).reshape(y.shape[0], -1, y.shape[1])


# ---------------------------------------------------------------------------------------------------------------------------
# the criterion
# ---------------------------------------------------------------------------------------------------------------------------
def judge(cid, out, ref, twin, branch, kappa=KAPPA):
    """out / ref / twin [B, P, C] fp64; asserts the criterion on every slice and prints the worst ratios"""
    assert out.shape == ref.shape == twin.shape, (cid, out.shape, ref.shape, twin.shape)
    assert torch.isfinite(out).all(), f"{cid}: non-finite output"
    B, P, C = out.shape
    G = SLICE_CH if C % SLICE_CH == 0 else C
    worst_r, worst_m, worst_k, bad = 0.0, 0.0, 0.0, []
    for b in range(B):
        for p0 in range(0, P, SLICE_POS):
            o, r, t = (z[b, p0:p0 + SLICE_POS].reshape(-1, C // G, G).transpose(0, 1).reshape(C // G, -1) for z in (out, ref, twin))
            eo, et, ed = o - r, t - r, o - t
            rms = lambda e: e.square().mean(1).sqrt()
            floor_r = rms(et) + U * rms(r)
            lim_r = RHO * rms(et) + U * rms(r)
            lim_m = RHO_MAX * et.abs().amax(1) + U * r.abs().amax(1)
            lim_k = kappa * rms(et) + U * rms(r)
            ratio_r = rms(eo) / floor_r
            ratio_m = eo.abs().amax(1) / (et.abs().amax(1) + U * r.abs().amax(1))
            ratio_k = rms(ed) / floor_r
            worst_r, worst_m = max(worst_r, ratio_r.max().item()), max(worst_m, ratio_m.max().item())
            worst_k = max(worst_k, ratio_k.max().item())
            for gi in torch.nonzero((rms(eo) > lim_r) | (eo.abs().amax(1) > lim_m) | (rms(ed) > lim_k)).flatten().tolist():
                bad.append(f"item {b} positions {p0}+ channels {gi * G}-{gi * G + G - 1}: rms ratio {ratio_r[gi].item():.2f} "
                           f"max ratio {ratio_m[gi].item():.2f} out-twin ratio {ratio_k[gi].item():.2f} (limit {kappa})")
    rel = (twin - ref).square().mean().sqrt().item() / max(ref.square().mean().sqrt().item(), 1e-300)
    print(f"[module] {cid:44s} {branch:34s} rms ratio {worst_r:5.2f}  max ratio {worst_m:5.2f}  out-twin ratio {worst_k:5.2f}  "
          f"twin rel rms {rel:.2e}")
    assert not bad, f"{cid}: {len(bad)} slices out of bound, e.g. " + "; ".join(bad[:4])


# ---------------------------------------------------------------------------------------------------------------------------
# fixtures: the full-size owners (emb slots and tables are theirs)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def unet2d():
    om = _unet_classes()
    return build(om.UNetModel2D_Next, dict(UNET2D, parts=["global", "data"]), DEV)


@pytest.fixture(scope="module")
def unet0d():
    om = _unet_classes()
    return build(om.UNetModel0D_Next, dict(UNET0D, parts=["global", "data"]), DEV)


def sd64(module, prefix="m"):
    return {f"{prefix}.{k}": v.detach().double().cpu() for k, v in module.state_dict().items()}


def round_weights(sd):
    return {k: bf(v) if v.dim() >= 2 else v for k, v in sd.items()}


def find_block(net, cls, pred, nth):
    hits = [(i, blk[0]) for i, blk in enumerate(net.data_blocks) if isinstance(blk[0], cls) and pred(blk[0])]
    assert hits, "no such block"
    return hits[nth]


def split_input(x, pair):
    """x [B, ..., C] on the device -> the block's input: x itself, or the pair (h, skip) that stands for it"""
    return (x[..., :pair[0]].contiguous(), x[..., pair[0]:].contiguous()) if pair else x


def pair_of(walk, m):
    return next(p for mm, _, _, _, p in walk if mm is m)


# ---------------------------------------------------------------------------------------------------------------------------
# one runner per module kind: each returns (out, ref, twin) as [B, P, C] fp64 and the branch it took
# ---------------------------------------------------------------------------------------------------------------------------
def t_emb_input(B, seed):
    ts = torch.randint(1, 1000, (B,), generator=gen(seed))
    return O().timestep_embedding(ts, 320)


def run_res(c, unet2d):
    om = _unet_classes()
    B, H, W = c["B"], c["H"], c["W"]
    if "idx" in c:
        idx, blk = c["idx"], unet2d.data_blocks[c["idx"]][0]
    else:
        idx, blk = find_block(unet2d, om.ResBlock, lambda m: (m.channels, m.out_channels) == (c["cin"], c["cout"]), c["nth"])
    pair = pair_of(walk_2d(unet2d, 1, 64, 64), blk)
    x = act_input(B, H * W, blk.channels, seed=idx * 7 + H)
    sd = sd64(blk)
    owner = {f"t.time_embed.{k}": v.detach().double().cpu() for k, v in unet2d.time_embed.state_dict().items()}
    t_emb = t_emb_input(B, idx)
    with torch.no_grad():
        xin = split_input(nhwc(x.to(DEV), B, H, W), pair)
        if c["emb"] == "table":
            emb_arg = unet2d.embed_table(t_emb.to(DEV))
        else:
            emb32 = unet2d.time_embedding(t_emb.to(DEV))
            emb_arg = unet2d.embed_all(emb32) if c["emb"] == "all" else emb32
        out = blk(xin, emb_arg)
    x64 = to_nchw64(x.view(B, H, W, -1))
    if c["emb"] == "table":     # the sinusoid in: the owner's time MLP (its first two GEMMs round to bf16), then the table
        ref = O().resblock(sd, "m", x64, O().time_embed(owner, "t", t_emb.double()))
        emb_tw = O().time_embed(round_weights(owner), "t", t_emb.double(), rounding("t_emb", "h"))
        twin = O().resblock(round_weights(sd), "m", x64, emb_tw, rounding("gn1", "emb_act", "conv1", "gn2", "out"))
    else:                       # the fp32 embedding the product was given (the time MLP has its own row)
        e = emb32.double().cpu()
        ref = O().resblock(sd, "m", x64, e)
        twin = O().resblock(round_weights(sd), "m", x64, e, rounding("gn1", "conv1", "gn2", "out"))
    if isinstance(emb_arg, om.EmbTable) == (c["emb"] != "emb"):       # what the block was given: a table, or the embedding
        REACHED.add(("emb", c["emb"]))
    if "idx" in c:
        REACHED.add(("res_slot", idx))
    REACHED.add(("skip", "pair" if pair else ("conv" if blk.packed()["has_skip"] else "identity")))
    return from_nchw(out.double().cpu().permute(0, 3, 1, 2)), from_nchw(ref), from_nchw(twin), f"data_blocks.{idx} emb {c['emb']}"


def st_module(C, heads, seed_key):
    from lib.model_zoo.attention import SpatialTransformer
    with torch.device("meta"):
        m = SpatialTransformer(C, heads, C // heads, context_dim=768)
    m = m.to_empty(device=DEV)
    fill_weights(m, seed_key + ".")
    return m.eval()


def st_twin_sd(sd, C, fold):
    """weights as the product stores them: bf16, and bf16(W gamma) / gamma where a LayerNorm is folded into the projection"""
    tw = round_weights(sd)
    if fold:
        t = "m.transformer_blocks.0"
        for w, n in ((".attn1.to_q", "norm1"), (".attn1.to_k", "norm1"), (".attn1.to_v", "norm1"), (".attn2.to_q", "norm2"),
                     (".ff.net.0.proj", "norm3")):
            g = sd[f"{t}.{n}.weight"]
            tw[f"{t}{w}.weight"] = bf(sd[f"{t}{w}.weight"] * g[None, :]) / g[None, :]
    return tw


ST_ROUND_COMMON = ("gn", "proj_in", "attn1", "attn2", "ff", "ff_hidden", "q", "k", "v", "p", "o")


def run_st(c):
    from lib.model_zoo.attention import ln_fold_fits
    B, H, W, C, L = c["B"], c["H"], c["W"], c["C"], c["L"]
    fold = ln_fold_fits(C, B, H, W)
    ragged = (H * W) % 8 != 0
    n_ctx = 2 if c["mix"] else 1
    mods = [st_module(C, c["heads"], f"st{C}.{i}") for i in range(n_ctx)]
    for m in mods:
        with torch.no_grad():
            m.proj_in.bias += c["tok_mean"]
        m.invalidate_packed()
    x = act_input(B, H * W, C, seed=C + H * 3 + L)
    Ls = (L, 257) if c["mix"] else (L,)
    # contexts share a component across their tokens (as encoder outputs do), so P V is not a mean of independent rows that
    # shrinks with L, and a weight given to the zero pad rows past L shows
    ctx = [(torch.randn(B, l, 768, generator=gen(C + l + i)) * 0.5 + torch.randn(B, 1, 768, generator=gen(C + l + i + 1))).to(torch.bfloat16)
           for i, l in enumerate(Ls)]
    with torch.no_grad():
        xd = nhwc(x.to(DEV), B, H, W)
        if c["mix"]:
            r1, r2 = c["mix"]
            acc = mods[0](xd, ctx[0].to(DEV), ratio=r1)
            out = mods[1](xd, ctx[1].to(DEV), ratio=r2, acc=acc)
        else:
            out = mods[0](xd, ctx[0].to(DEV))
    x64 = to_nchw64(x.view(B, H, W, -1))
    names = ST_ROUND_COMMON + (() if fold else ("ln1", "ln2", "ln3"))
    refs, twins = [], []
    for m, cx in zip(mods, ctx):
        sd = sd64(m)
        refs.append(torch.cat([O().spatial_transformer(sd, "m", x64[b:b + 1], cx[b:b + 1].double(), c["heads"]) for b in range(B)]))
        tw = st_twin_sd(sd, C, fold)
        rnd = rounding(*(names if c["mix"] else names + ("out",)))
        twins.append(torch.cat([O().spatial_transformer(tw, "m", x64[b:b + 1], cx[b:b + 1].double(), c["heads"], rnd)
                                for b in range(B)]))
    if c["mix"]:
        r1, r2 = c["mix"]
        ref = r1 * refs[0] + r2 * refs[1]                                    # the context mixing of apply_model (vd.py:391-396)
        acc = bf(x64 + r1 * (twins[0] - x64))                                # proj_out epilogues: h + r1 delta1, then + r2 delta2
        twin = bf(acc + r2 * (twins[1] - x64))
        REACHED.add(("mix",))
    else:
        ref, twin = refs[0], twins[0]
    REACHED.add(("ln", "fold" if fold else "plain"))
    REACHED.add(("self", "ragged" if ragged else "aligned"))
    REACHED.add(("ctx_pad", any(l % 8 for l in Ls)))
    branch = f"{'folded' if fold else 'plain'} LN, {'ragged' if ragged else 'aligned'}, L {'/'.join(map(str, Ls))}"
    return from_nchw(out.double().cpu().permute(0, 3, 1, 2)), from_nchw(ref), from_nchw(twin), branch


def run_conv(c, unet2d):
    """ConvIn, Downsample, Upsample and OutHead of the full-size UNet"""
    om = _unet_classes()
    from lib.model_zoo.diffusion_utils import upsample_fold_enabled
    B, H, W, C, k = c["B"], c["H"], c["W"], c["C"], c["kind"]
    cls = {"convin": om.ConvIn, "down": om.Downsample, "up": om.Upsample, "outhead": om.OutHead}[k]
    chan = {om.ConvIn: lambda m: m.in_channels, om.Downsample: lambda m: m.channels, om.Upsample: lambda m: m.channels,
            om.OutHead: lambda m: getattr(m, "0").num_channels}[cls]
    idx, m = find_block(unet2d, cls, lambda m: chan(m) == C, 0)
    sd = sd64(m)
    tw = round_weights(sd)
    if k == "convin":
        x = (torch.randn(B, H, W, C, generator=gen(H)) * 1.5).to(torch.bfloat16).float()     # bf16-exact fp32 latent
        with torch.no_grad():
            out = m(x.to(DEV))
        x64 = x.double().permute(0, 3, 1, 2)
        ref, twin = O().conv_in(sd, "m", x64), bf(O().conv_in(tw, "m", x64))
        branch = "im2col + GEMM"
    else:
        x = act_input(B, H * W, C, seed=C + H)
        with torch.no_grad():
            out = m(nhwc(x.to(DEV), B, H, W))
        x64 = to_nchw64(x.view(B, H, W, -1))
        if k == "down":
            ref, twin = O().downsample(sd, "m", x64), bf(O().downsample(tw, "m", x64))
            branch = "conv mode 1"
        elif k == "up":
            ref, twin = O().upsample(sd, "m", x64), bf(O().upsample(tw, "m", x64))
            fold = upsample_fold_enabled(B * H * W, m.out_channels)
            REACHED.add(("up", "fold" if fold else "plain"))
            branch = "folded" if fold else "upsample2x + conv"
        else:
            ref, twin = O().out_head(sd, "m", x64), O().out_head(tw, "m", x64, rounding("gn"))
            branch = "fp32 out"
    return from_nchw(out.double().cpu().permute(0, 3, 1, 2)), from_nchw(ref), from_nchw(twin), f"data_blocks.{idx} {branch}"


def run_time(c, unet2d):
    B = c["B"]
    t_emb = t_emb_input(B, 5)
    sd = {f"t.time_embed.{k}": v.detach().double().cpu() for k, v in unet2d.time_embed.state_dict().items()}
    with torch.no_grad():
        out = unet2d.time_embedding(t_emb.to(DEV))
    ref = O().time_embed(sd, "t", t_emb.double())
    twin = O().time_embed(round_weights(sd), "t", t_emb.double())
    return out.double().cpu()[:, None], ref[:, None], twin[:, None], "linear_small x2, fp32"


def md(y, B):
    """the oracle's [B, C, s, 1] -> [B, s, C]"""
    return y.permute(0, 2, 3, 1).reshape(B, y.shape[2], y.shape[1])


def run_0d(c, unet0d):
    om = _unet_classes()
    B, k = c["B"], c["kind"]
    if k == "fc":
        if "idx" in c:
            idx, m = c["idx"], unet0d.data_blocks[c["idx"]][0]
        else:
            idx, m = find_block(unet0d, om.FCBlock_MultiDim, lambda m: (m.channels_multidim[0], m.out_channels_multidim[0]) ==
                                (c["cin"], c["cout"]), 0)
        pair = pair_of(walk_0d(unet0d), m)
        x = act_input(B, 4, m.channels_multidim[0], seed=idx)
        t_emb = t_emb_input(B, idx)
        sd, owner = sd64(m), {f"t.time_embed.{k}": v.detach().double().cpu() for k, v in unet0d.time_embed.state_dict().items()}
        with torch.no_grad():
            xin = split_input(x.to(DEV).view(B, 4, 1, -1), pair)
            if c["emb"] == "table":
                emb_arg = unet0d.embed_table(t_emb.to(DEV))
            else:
                emb_arg = unet0d.time_embedding(t_emb.to(DEV))
            out = m(xin, emb_arg)
        x64 = x.double().view(B, 4, 1, -1).permute(0, 3, 1, 2)
        names = ("gn1_hat", "gn1", "conv1", "gn2_hat", "gn2", "out")
        if c["emb"] == "table":
            ref = O().fcblock(sd, "m", x64, O().time_embed(owner, "t", t_emb.double()))
            emb_tw = O().time_embed(round_weights(owner), "t", t_emb.double(), rounding("t_emb", "h"))
            twin = O().fcblock(round_weights(sd), "m", x64, emb_tw, rounding("emb_act", *names))
        else:
            e = emb_arg.double().cpu()
            ref = O().fcblock(sd, "m", x64, e)
            twin = O().fcblock(round_weights(sd), "m", x64, e, rounding(*names))
        REACHED.add(("fc_skip", "pair" if pair else ("conv" if m.packed()["has_skip"] else "identity")))
        if isinstance(emb_arg, om.EmbTable) == (c["emb"] == "table"):
            REACHED.add(("fc_emb", c["emb"]))
        if "idx" in c:
            REACHED.add(("fc_slot", idx))
        return md(out.double().cpu().permute(0, 3, 1, 2), B), md(ref, B), md(twin, B), f"data_blocks.{idx} emb {c['emb']}"
    if k == "lin":
        idx, m = find_block(unet0d, om.Linear_MultiDim, lambda m: (tuple(m.in_features_multidim), tuple(m.out_features_multidim)) ==
                            (c["fin"], c["fout"]), 0)
        sd = sd64(m)
        if len(c["fin"]) == 1:
            x = (torch.randn(B, 768, generator=gen(3))).to(torch.bfloat16).float()      # the fp32 latent, bf16-exact
            xin, x64 = x.to(DEV), x.double()
        else:
            xb = act_input(B, 4, c["fin"][0], seed=idx)
            xin, x64 = xb.to(DEV).view(B, 4, 1, -1), xb.double().view(B, 4, 1, -1).permute(0, 3, 1, 2)
        with torch.no_grad():
            out = m(xin)
        ref, twin = O().linear_md(sd, "m", x64), bf(O().linear_md(round_weights(sd), "m", x64))
        return md(out.double().cpu().permute(0, 3, 1, 2), B), md(ref, B), md(twin, B), f"data_blocks.{idx}"
    idx, m = find_block(unet0d, om.OutHead0D, lambda m: True, 0)
    sd = sd64(m)
    x = act_input(B, 4, c["C"], seed=9)
    with torch.no_grad():
        out = m(x.to(DEV).view(B, 4, 1, -1))
    x64 = x.double().view(B, 4, 1, -1).permute(0, 3, 1, 2)
    ref, twin = O().out_head0d(sd, "m", x64), O().out_head0d(round_weights(sd), "m", x64, rounding("gn"))
    return out.double().cpu()[:, None], ref[:, None], twin[:, None], f"data_blocks.{idx} fp32 out"


def vae_module(c):
    from lib.model_zoo import autokl_modules as ak
    k = c["kind"]
    if k == "vres":
        return build(ak.ResnetBlock, dict(in_channels=c["cin"], out_channels=c["cout"], dropout=0.0, temb_channels=0), DEV)
    if k == "vattn":
        return build(ak.AttnBlock, dict(in_channels=c["C"]), DEV)
    if k == "vup":
        return build(ak.Upsample, dict(in_channels=c["C"], with_conv=True), DEV)
    return build(ak.Downsample, dict(in_channels=c["C"], with_conv=True), DEV)


def run_vae(c):
    from lib.model_zoo.diffusion_utils import upsample_fold_enabled
    B, H, W, k = c["B"], c["H"], c["W"], c["kind"]
    m = vae_module(c)
    cin = c.get("cin", c.get("C"))
    x = act_input(B, H * W, cin, seed=cin + H, scale=8.0)
    with torch.no_grad():
        out = m(nhwc(x.to(DEV), B, H, W))
    x64 = to_nchw64(x.view(B, H, W, -1))
    sd = sd64(m)
    tw = round_weights(sd)
    if k == "vres":
        ref, twin = O().vae_resnet(sd, "m", x64), O().vae_resnet(tw, "m", x64, rounding("gn1", "conv1", "gn2", "out"))
        branch = "nin_shortcut" if m.packed()["has_skip"] else "identity"
        REACHED.add(("vres", branch))
    elif k == "vattn":
        ref = O().vae_attn(sd, "m", x64)
        twin = O().vae_attn(tw, "m", x64, rounding("gn", "q", "k", "s", "p", "v", "o", "out"))
        branch = "S, softmax_rows, P v + b_v"
    elif k == "vup":
        ref, twin = O().upsample(sd, "m", x64), bf(O().upsample(tw, "m", x64))
        fold = upsample_fold_enabled(B * H * W, c["C"])
        REACHED.add(("vup", "fold" if fold else "plain"))
        branch = "folded" if fold else "upsample2x + conv"
    else:
        ref, twin = O().vae_downsample(sd, "m", x64), bf(O().vae_downsample(tw, "m", x64))
        branch = "conv mode 2"
    return from_nchw(out.double().cpu().permute(0, 3, 1, 2)), from_nchw(ref), from_nchw(twin), branch


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_module_case(case, request):
    k = case["kind"]
    with torch.no_grad():
        if k == "res":
            got = run_res(case, request.getfixturevalue("unet2d"))
        elif k == "st":
            got = run_st(case)
        elif k in ("convin", "down", "up", "outhead"):
            got = run_conv(case, request.getfixturevalue("unet2d"))
        elif k == "time":
            got = run_time(case, request.getfixturevalue("unet2d"))
        elif k in ("fc", "lin", "out0d"):
            got = run_0d(case, request.getfixturevalue("unet0d"))
        else:
            got = run_vae(case)
    RAN.add(case["id"])
    judge(case["id"], *got, kappa=case.get("kappa", KAPPA))


# ---------------------------------------------------------------------------------------------------------------------------
def test_twin_with_identity_rounding_is_the_oracle():
    """the hooked paths (softmax as exp / sum, the GroupNorm affine after normalising, b_v after P v) equal the oracle's own
    evaluation to 1e-12 when the hook rounds nothing"""
    from lib.model_zoo import attention as at
    from lib.model_zoo import autokl_modules as ak
    om = _unet_classes()
    g = gen(0)
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    m = build(at.SpatialTransformer, dict(in_channels=64, n_heads=8, d_head=8, context_dim=768), "cpu")
    sd = sd64(m)
    x, c = torch.randn(2, 64, 4, 6, generator=g, dtype=torch.float64), torch.randn(2, 77, 768, generator=g, dtype=torch.float64)
    assert rel(O().spatial_transformer(sd, "m", x, c, 8, identity), O().spatial_transformer(sd, "m", x, c, 8)) < 1e-12
    m = build(om.FCBlock_MultiDim, dict(channels=[64, 4, 1], emb_channels=128, dropout=0, out_channels=[96, 4, 1]), "cpu")
    sd, x, e = sd64(m), torch.randn(2, 64, 4, 1, generator=g, dtype=torch.float64), torch.randn(2, 128, generator=g, dtype=torch.float64)
    assert rel(O().fcblock(sd, "m", x, e, identity), O().fcblock(sd, "m", x, e)) < 1e-12
    m = build(om.ResBlock, dict(channels=64, emb_channels=128, dropout=0, out_channels=96), "cpu")
    sd, x = sd64(m), torch.randn(2, 64, 6, 5, generator=g, dtype=torch.float64)
    assert rel(O().resblock(sd, "m", x, e, identity), O().resblock(sd, "m", x, e)) < 1e-12
    m = build(ak.AttnBlock, dict(in_channels=64), "cpu")
    sd, x = sd64(m), torch.randn(2, 64, 6, 5, generator=g, dtype=torch.float64) * 30
    assert rel(O().vae_attn(sd, "m", x, identity), O().vae_attn(sd, "m", x)) < 1e-12
    m = build(ak.ResnetBlock, dict(in_channels=64, out_channels=32, dropout=0.0, temb_channels=0), "cpu")
    sd = sd64(m)
    assert rel(O().vae_resnet(sd, "m", x, identity), O().vae_resnet(sd, "m", x)) < 1e-12


def full_size_signatures():
    """the configuration signature of every layer module of the full-size models at the driven shapes, and the modules walked"""
    om = _unet_classes()
    from lib.model_zoo import autokl_modules as ak
    u2 = build(om.UNetModel2D_Next, dict(UNET2D), "meta")
    u0 = build(om.UNetModel0D_Next, dict(UNET0D), "meta")
    enc, dec = build(ak.Encoder, VAE, "meta"), build(ak.Decoder, VAE, "meta")
    walked = []
    for B, H, W, levels in DRIVES_2D:
        walked += walk_2d(u2, B, H, W, levels)
    walked += walk_0d(u0) + walk_vae(enc, dec)
    sigs = {s for m, B, H, W, pair in walked for s in signatures(m, B, H, W, pair)}
    layer_classes = (om.ResBlock, om.ConvIn, om.Downsample, om.Upsample, om.OutHead, om.FCBlock_MultiDim, om.Linear_MultiDim,
                     om.OutHead0D, om.SpatialTransformer, ak.ResnetBlock, ak.AttnBlock, ak.Upsample, ak.Downsample)
    inner = {id(getattr(m, "2")) for m in u0.modules() if isinstance(m, om.OutHead0D)}     # (its Linear_MultiDim is its own)
    every = {id(m) for net in (u2, u0, enc, dec) for m in net.modules() if isinstance(m, layer_classes)} - inner
    return sigs, every, {id(m) for m, *_ in walked}


def test_every_configuration_has_a_case():
    """every layer module of the full-size 2-D UNet, 0-D diffuser and VAE, at every driven shape, has a row in CASES (a new
    module shape cannot land untested), and the walk reached every layer module the models hold"""
    sigs, every, walked = full_size_signatures()
    assert every == walked, f"{len(every - walked)} layer modules the walk does not reach"
    have = {case_signature(c) for c in CASES}
    missing = sorted(sigs - have, key=str)
    assert not missing, f"{len(missing)} configurations without a case, e.g. {missing[:6]}"
    print(f"[module] {len(sigs)} configurations of the full-size models, {len(CASES)} cases")


@pytest.mark.gpu
def test_every_path_reached():
    """the case tests took every branch of the layer code, as the code's own predicates decide it"""
    if RAN != {c["id"] for c in CASES}:
        pytest.skip("runs after the whole case table")
    want = {("emb", "table"), ("emb", "emb"), ("emb", "all"), ("skip", "identity"), ("skip", "conv"), ("skip", "pair"),
            ("ln", "fold"), ("ln", "plain"), ("self", "ragged"), ("self", "aligned"), ("ctx_pad", True), ("mix",),
            ("up", "fold"), ("up", "plain"), ("fc_skip", "identity"), ("fc_skip", "conv"), ("fc_skip", "pair"),
            ("fc_emb", "table"), ("fc_emb", "emb"), ("vres", "identity"), ("vres", "nin_shortcut"), ("vup", "fold"),
            ("vup", "plain")}
    want |= {("res_slot", i) for kind, i, _ in O().unet_layout() if kind == "res"}
    want |= {("fc_slot", i) for kind, i in O().unet0d_layout() if kind == "fc"}
    assert want <= REACHED, f"not reached: {sorted(want - REACHED, key=str)}"
