"""CPU oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

A plain fp32 torch-on-CPU restatement of the Versatile-Diffusion sampling hot path, written as pure
functions over a state_dict that uses the reference's checkpoint key names.  Each
function cites the reference file:line it follows (paths relative to /root/reference).  It is pinned
against the unmodified reference itself: oracle/make_golden.py imports the reference (under the shims
of oracle/ref_shims.py), runs it on seeded inputs and commits the outputs to tests/golden/;
tests/test_oracle.py checks this restatement against those fixtures, and against the live reference
when /root/reference exists.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference leg may import this module.

CLIP: the arithmetic of the context encoders lives in the third-party `transformers` package
(reference pins transformers==4.24.0, requirements.txt:12; call sites lib/model_zoo/clip.py:53-62 and
:88-101).  `clip_text_encode` / `clip_image_encode` restate the published CLIP ViT-L/14 algorithm
(pre-LN transformer, quick_gelu, causal text mask) and are pinned against `transformers.CLIPModel`
(version in this image: 5.5.0) on random-init weights — the reference holds no CLIP test vectors,
so CLIP parity is pinned to that implementation, not to pretrained outputs.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------
# schedules
# ------------------------------------------------------------------------------------------------
def make_beta_schedule(n_timestep=1000, linear_start=0.00085, linear_end=0.012):
    """'linear' branch of make_beta_schedule, lib/model_zoo/diffusion_utils.py:8-13 (fp64)."""
    return (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()


def ddpm_schedule(n_timestep=1000, linear_start=0.00085, linear_end=0.012):
    """VD_v2_0.register_schedule, lib/model_zoo/vd.py:127-162: fp64 numpy -> fp32 buffers."""
    betas = make_beta_schedule(n_timestep, linear_start, linear_end)
    alphas = 1.0 - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1.0, ac[:-1])
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)
    return {
        "betas": f32(betas), "alphas_cumprod": f32(ac), "alphas_cumprod_prev": f32(ac_prev),
        "sqrt_alphas_cumprod": f32(np.sqrt(ac)), "sqrt_one_minus_alphas_cumprod": f32(np.sqrt(1.0 - ac)),
    }


def make_ddim_timesteps(num_ddim, num_ddpm=1000):
    """'uniform' branch, diffusion_utils.py:32-46: range(0, T, T//S) + 1."""
    c = num_ddpm // num_ddim
    return np.asarray(list(range(0, num_ddpm, c))) + 1


def ddim_schedule(alphas_cumprod, num_ddim, eta=0.0, timesteps=None):
    """DDIMSampler.make_schedule + make_ddim_sampling_parameters, ddim.py:23-56, diffusion_utils.py:48-59.
    alphas_cumprod: fp32 tensor (the model buffer). Returns fp32 python lists per DDIM index, with the
    same dtype walk as the reference: alphas fp32 tensor; alphas_prev fp64 ndarray built from fp32
    values; sigmas = eta*sqrt(...) in fp64; sqrt(1-alphas) on the fp32 tensor.  timesteps: the grid
    (default DDIM's uniform one of num_ddim steps)."""
    ts = make_ddim_timesteps(num_ddim, alphas_cumprod.shape[0]) if timesteps is None else np.asarray(timesteps)
    ac = alphas_cumprod.cpu()
    alphas = ac[ts]                                                       # fp32 tensor
    alphas_prev = np.asarray([ac[0]] + ac[ts[:-1]].tolist())              # fp64 ndarray of fp32 values
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas.double().numpy()) * (1 - alphas.double().numpy() / alphas_prev))
    sqrt_1m = np.sqrt(1.0 - alphas.numpy())                               # fp32
    return {
        "timesteps": ts,
        "alphas": alphas.numpy().astype(np.float32),
        "alphas_prev": alphas_prev.astype(np.float32),                    # torch.full(..., dtype=fp32) cast
        "sigmas": np.asarray(sigmas).astype(np.float32),
        "sqrt_one_minus_alphas": sqrt_1m.astype(np.float32),
    }


def timestep_embedding(timesteps, dim, max_period=10000):
    """diffusion_utils.py:131-151 — [cos | sin], fp32."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    args = timesteps[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


# ------------------------------------------------------------------------------------------------
# UNet building blocks
# ------------------------------------------------------------------------------------------------
def _gn(x, sd, p, eps):
    return F.group_norm(x, 32, sd[p + ".weight"], sd[p + ".bias"], eps)


def _identity(name, t):
    return t


# Rounding hook.  Every block function below takes rnd(name, tensor) -> tensor, applied to the named intermediate where the
# reference's evaluation passes it on; the default is the identity, so the functions compute the reference unchanged.  A test
# passes a hook that rounds the activations a lower-precision implementation stores (tests/test_module_coverage_gpu.py).  Names:
#   resblock / vae_resnet:  "gn1" (SiLU(GroupNorm(x))), "emb_act" (SiLU(emb)), "conv1" (conv1 + emb), "gn2", "out"
#   cross_attention:        "q", "k", "v", "p" (the softmax numerator weights exp(s - max), see below), "o" (heads merged)
#   spatial_transformer:    "gn", "proj_in", "ln1" / "ln2" / "ln3", "attn1" / "attn2" (tokens after each residual),
#                           "ff_hidden" (GEGLU output), "ff" (tokens after the feed-forward residual), "out"
#   fcblock:                "gn1_hat" / "gn2_hat" (GroupNorm before its affine), "gn1" / "gn2", "conv1", "out"
#   vae_attn:               "gn", "q", "k", "s" (q k^T), "p" (softmax), "v" (without its bias), "o" (P v + b_v), "out"
#   time_embed:             "t_emb", "h" (SiLU of the first linear), "out"
# cross_attention and vae_attn evaluate the softmax as exp(s - max) / sum exp(s - max) when a hook is given, so that "p" can
# round the numerator's weights alone; fcblock then applies the GroupNorm affine after normalising.  Both equal the default
# path up to fp64 reordering.
def resblock(sd, p, x, emb, rnd=None):
    """ResBlock._forward (non-updown, use_scale_shift_norm=False), openaimodel.py:254-274; GN eps 1e-5."""
    r = rnd or _identity
    h = F.conv2d(r("gn1", F.silu(_gn(x, sd, p + ".in_layers.0", 1e-5))), sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"],
                 padding=1)
    e = F.linear(r("emb_act", F.silu(emb)), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])
    h = r("conv1", h + e[:, :, None, None])
    h = F.conv2d(r("gn2", F.silu(_gn(h, sd, p + ".out_layers.0", 1e-5))), sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"],
                 padding=1)
    if (p + ".skip_connection.weight") in sd:
        x = F.conv2d(x, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    return r("out", x + h)


def cross_attention(sd, p, x, context, heads, rnd=None, hook=None):
    """CrossAttention.forward, attention.py:170-193 (no mask on this path).  hook(probs [b, heads, n, L], is_cross) -> the
    softmax probabilities that weight V, for the oracles that read or edit the attention maps (SAG, Prompt-to-Prompt)."""
    assert rnd is None or hook is None
    r = rnd or _identity
    cross = context is not None
    context = x if context is None else context
    q = r("q", F.linear(x, sd[p + ".to_q.weight"]))
    k = r("k", F.linear(context, sd[p + ".to_k.weight"]))
    v = r("v", F.linear(context, sd[p + ".to_v.weight"]))
    b, n, c = q.shape
    d = c // heads
    split = lambda t: t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3)
    q, k, v = split(q), split(k), split(v)
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * d ** -0.5
    if rnd is None:
        probs = sim.softmax(dim=-1)
        if hook is not None:
            probs = hook(probs, cross)
        out = torch.einsum("bhij,bhjd->bhid", probs, v)
    else:
        w = (sim - sim.amax(-1, keepdim=True)).exp()
        out = torch.einsum("bhij,bhjd->bhid", r("p", w), v) / w.sum(-1, keepdim=True)
    out = r("o", out.permute(0, 2, 1, 3).reshape(b, n, c))
    return F.linear(out, sd[p + ".to_out.0.weight"], sd[p + ".to_out.0.bias"])


def spatial_transformer(sd, p, x, context, heads, rnd=None, hook=None):
    """SpatialTransformer.forward -> BasicTransformerBlock._forward (depth 1), attention.py:214-218,255-266."""
    r = rnd or _identity
    b, c, h, w = x.shape
    x_in = x
    x = r("gn", _gn(x, sd, p + ".norm", 1e-6))
    x = r("proj_in", F.conv2d(x, sd[p + ".proj_in.weight"], sd[p + ".proj_in.bias"]))
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, c)
    t = p + ".transformer_blocks.0"
    ln = lambda y, n: r("ln" + n[-1], F.layer_norm(y, (c,), sd[f"{t}.{n}.weight"], sd[f"{t}.{n}.bias"], 1e-5))
    x = r("attn1", cross_attention(sd, t + ".attn1", ln(x, "norm1"), None, heads, rnd, hook) + x)
    x = r("attn2", cross_attention(sd, t + ".attn2", ln(x, "norm2"), context, heads, rnd, hook) + x)
    hdn = F.linear(ln(x, "norm3"), sd[t + ".ff.net.0.proj.weight"], sd[t + ".ff.net.0.proj.bias"])
    val, gate = hdn.chunk(2, dim=-1)                       # GEGLU, attention.py:42-44 (erf gelu)
    x = r("ff", F.linear(r("ff_hidden", val * F.gelu(gate)), sd[t + ".ff.net.2.weight"], sd[t + ".ff.net.2.bias"]) + x)
    x = x.reshape(b, h, w, c).permute(0, 3, 1, 2)
    x = F.conv2d(x, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    return r("out", x + x_in)


def time_embed(sd, p, t_emb, rnd=None):
    """The time_embed MLP, openaimodel.py:2629-2633: Linear -> SiLU -> Linear on the sinusoid."""
    r = rnd or _identity
    h = r("h", F.silu(F.linear(r("t_emb", t_emb), sd[p + ".time_embed.0.weight"], sd[p + ".time_embed.0.bias"])))
    return r("out", F.linear(h, sd[p + ".time_embed.2.weight"], sd[p + ".time_embed.2.bias"]))


def conv_in(sd, p, x):
    """data_blocks.0: conv3x3 pad 1 on the latent, openaimodel.py:2664."""
    return F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], padding=1)


def downsample(sd, p, x):
    """Downsample.op: conv3x3 stride 2 pad 1, openaimodel.py:150-159."""
    return F.conv2d(x, sd[p + ".op.weight"], sd[p + ".op.bias"], stride=2, padding=1)


def upsample(sd, p, x):
    """Upsample (openaimodel.py:107-117) and the VAE's (autokl_modules.py:38-47): nearest x2 then conv3x3 pad 1."""
    x = F.interpolate(x, scale_factor=2, mode="nearest")
    return F.conv2d(x, sd[p + ".conv.weight"], sd[p + ".conv.bias"], padding=1)


def out_head(sd, p, x, rnd=None):
    """GN -> SiLU -> conv3x3, openaimodel.py:2732-2737."""
    r = rnd or _identity
    return F.conv2d(r("gn", F.silu(_gn(x, sd, p + ".0", 1e-5))), sd[p + ".2.weight"], sd[p + ".2.bias"], padding=1)


def linear_md(sd, p, x, second_dim=4):
    """Linear_MultiDim (openaimodel.py:2275-2293): nn.Linear over the flattened feature, viewed back as [B, C, second_dim, 1]."""
    b = x.shape[0]
    return F.linear(x.reshape(b, -1), sd[p + ".weight"], sd[p + ".bias"]).view(b, -1, second_dim, 1)


def out_head0d(sd, p, x, rnd=None):
    """GroupNorm32(C) -> SiLU -> Linear_MultiDim([C, s, 1] -> [768]), openaimodel.py:2957-2962."""
    r = rnd or _identity
    h = r("gn", F.silu(_gn(x, sd, p + ".0", 1e-5)))
    return F.linear(h.reshape(x.shape[0], -1), sd[p + ".2.weight"], sd[p + ".2.bias"])


def unet_layout(model_channels=320, channel_mult=(1, 2, 4, 4), num_res_blocks=(2, 2, 2, 2),
                attention_resolutions=(4, 2, 1), num_heads=8):
    """The layer walk of UNetModel2D_Next.__init__, openaimodel.py:2664-2740: a list of
    ('conv_in'|'res'|'ctx'|'down'|'up'|'out'|'save'|'load', data_idx/ctx_idx, meta) in execution order."""
    ops, d, c = [], 0, 0
    ops.append(("conv_in", d, None)); d += 1
    ops.append(("save", None, None))
    ds = 1
    for level, mult in enumerate(channel_mult):
        for _ in range(num_res_blocks[level]):
            ops.append(("res", d, None)); d += 1
            if ds in attention_resolutions:
                ops.append(("ctx", c, None)); c += 1
            ops.append(("save", None, None))
        if level != len(channel_mult) - 1:
            ops.append(("down", d, None)); d += 1
            ops.append(("save", None, None))
            ds *= 2
    ops.append(("res", d, None)); d += 1
    ops.append(("ctx", c, None)); c += 1
    ops.append(("res", d, None)); d += 1
    for level, mult in list(enumerate(channel_mult))[::-1]:
        for _ in range(num_res_blocks[level] + 1):
            ops.append(("load", None, None))
            ops.append(("res", d, None)); d += 1
            if ds in attention_resolutions:
                ops.append(("ctx", c, None)); c += 1
        if level != 0:
            ops.append(("up", d, None)); d += 1
            ds //= 2
    ops.append(("out", d, None)); d += 1
    return ops


def fcblock(sd, p, x, emb, rnd=None):
    """FCBlock_MultiDim.forward -> FCBlock._forward, openaimodel.py:2134-2141, 2344-2354: the [B, C, s, 1] feature is flattened
    to C*s*1 channels of a 1x1 "image" (index c*s + si), GroupNorm32 (eps 1e-5) -> SiLU -> 1x1 conv, + SiLU->Linear(emb),
    GroupNorm32 -> SiLU -> 1x1 conv, + skip (identity or 1x1 conv); the result is viewed back as [B, Cout, s, 1]."""
    r = rnd or _identity
    b, _, sdim, _ = x.shape
    xf = x.reshape(b, -1, 1, 1)

    def gn_silu(y, q, n):
        if rnd is None:
            return F.silu(_gn(y, sd, q, 1e-5))
        y = r(n + "_hat", F.group_norm(y, 32, None, None, 1e-5))
        return r(n, F.silu(y * sd[q + ".weight"][:, None, None] + sd[q + ".bias"][:, None, None]))
    h = F.conv2d(gn_silu(xf, p + ".in_layers.0", "gn1"), sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"])
    e = F.linear(r("emb_act", F.silu(emb)), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])
    h = r("conv1", h + e[:, :, None, None])
    h = F.conv2d(gn_silu(h, p + ".out_layers.0", "gn2"), sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"])
    if (p + ".skip_connection.weight") in sd:
        xf = F.conv2d(xf, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    y = r("out", xf + h)
    return y.reshape(b, y.shape[1] // sdim, sdim, 1)


def unet0d_layout(channel_mult=(1, 2, 4, 4), num_noattn_blocks=(2, 2, 2, 2), with_attn=(True, True, True, False)):
    """The layer walk of UNetModel0D_Next.__init__, openaimodel.py:2885-2962: ('lin_in'|'fc'|'ctx'|'lin'|'out'|'save'|'load',
    data_idx / ctx_idx) in execution order."""
    ops, d, c = [], 0, 0
    ops.append(("lin_in", d)); d += 1
    ops.append(("save", None))
    for level in range(len(channel_mult)):
        for _ in range(num_noattn_blocks[level]):
            ops.append(("fc", d)); d += 1
            if with_attn[level]:
                ops.append(("ctx", c)); c += 1
            ops.append(("save", None))
        if level != len(channel_mult) - 1:
            ops.append(("lin", d)); d += 1
            ops.append(("save", None))
    ops.append(("fc", d)); d += 1
    ops.append(("ctx", c)); c += 1
    ops.append(("fc", d)); d += 1
    for level in list(range(len(channel_mult)))[::-1]:
        for _ in range(num_noattn_blocks[level] + 1):
            ops.append(("load", None))
            ops.append(("fc", d)); d += 1
            if with_attn[level]:
                ops.append(("ctx", c)); c += 1
        if level != 0:
            ops.append(("lin", d)); d += 1
    ops.append(("out", d)); d += 1
    return ops


def context_weights(ratios, n):
    """the mixing weights of n contexts: their ratios (None: equal) normalised to sum 1, fp64"""
    r = np.array([1.0] * n if ratios is None else ratios, dtype=np.float64)
    return r / r.sum()


def context_block(sd, idx, h, contexts, ratios, c_types, num_heads, hook_for=None):
    """context block idx of diffuser.<c_type> on h for every context; several contexts are mixed by context_weights
    (context_mixing 'attention', vd.py:383-395).  hook_for(j, idx) -> the attention hook of context j (cross_attention), or None."""
    r = context_weights(ratios, len(contexts))
    acc = None
    for j, (ct, c) in enumerate(zip(c_types, contexts)):
        hook = None if hook_for is None else hook_for(j, idx)
        hj = spatial_transformer(sd, f"diffuser.{ct}.context_blocks.{idx}.0", h, c, num_heads, hook=hook)
        if len(contexts) > 1:
            hj = hj * r[j]
        acc = hj if acc is None else acc + hj
    return acc


def apply_model_text(sd, x, timesteps, contexts, ratios=None, c_types=("text",), layout=None, model_channels=320,
                     second_dim=4, num_heads=8, time_from="image"):
    """VD_v2_0.apply_model / apply_model_multicontext (vd.py:330-455) for x_type = 'text': the 0-D diffuser's data blocks
    (Linear_MultiDim / FCBlock_MultiDim, openaimodel.py:2275-2354, 2885-2962) on a [B, 768] text latent, context blocks of
    diffuser[c_type] on the [B, C, second_dim, 1] feature (four "pixels").  time_embed comes from diffuser[global_layer_ptr]
    (= 'image' in vd_four_flow) for apply_model and from diffuser['text'] for the multicontext variant (vd.py:339, 415)."""
    layout = layout or unet0d_layout()
    D = "diffuser.text"
    T = f"diffuser.{time_from}"
    emb = time_embed(sd, T, timestep_embedding(timesteps, model_channels))
    hs, h = [], x
    for kind, idx in layout:
        p = f"{D}.data_blocks.{idx}.0"
        if kind in ("lin_in", "lin"):      # Linear_MultiDim([768] or [C, s, 1] -> [C, s, 1])
            h = linear_md(sd, p, h, second_dim)
        elif kind == "fc":
            h = fcblock(sd, p, h, emb)
        elif kind == "out":
            h = out_head0d(sd, p, h)
        elif kind == "ctx":
            h = context_block(sd, idx, h, contexts, ratios, c_types, num_heads)
        elif kind == "save":
            hs.append(h)
        elif kind == "load":
            h = torch.cat([h, hs.pop()], dim=1)
    return h


def apply_model(sd, x, timesteps, contexts, ratios=None, x_type="image", c_types=("text",), layout=None,
                model_channels=320, num_heads=8, hook_for=None):
    """VD_v2_0.apply_model (vd.py:330-381) when len(contexts)==1 and apply_model_multicontext +
    context_mixing 'attention' (vd.py:383-455) otherwise.  sd keys: diffuser.<type>.… ; the time
    embedding comes from diffuser.<x_type> (global_layer_ptr='image' == x_type on this path).
    hook_for(j, idx) -> the attention hook of context j in context block idx (see context_block)."""
    layout = layout or unet_layout(model_channels=model_channels, num_heads=num_heads)
    D = f"diffuser.{x_type}"
    emb = time_embed(sd, D, timestep_embedding(timesteps, model_channels))
    hs, h = [], x
    for kind, idx, _ in layout:
        p = f"{D}.data_blocks.{idx}.0"
        if kind == "conv_in":
            h = conv_in(sd, p, h)
        elif kind == "res":
            h = resblock(sd, p, h, emb)
        elif kind == "down":
            h = downsample(sd, p, h)
        elif kind == "up":
            h = upsample(sd, p, h)
        elif kind == "out":
            h = out_head(sd, p, h)
        elif kind == "ctx":
            h = context_block(sd, idx, h, contexts, ratios, c_types, num_heads, hook_for)
        elif kind == "save":
            hs.append(h)
        elif kind == "load":
            h = torch.cat([h, hs.pop()], dim=1)
    return h


def cfg_pass(model, sd, x, t, conds, unconds, pair, ratios=None, c_types=("text",), **kw):
    """model (apply_model or apply_model_text) on x alone -> (None, e_c), or on the CFG batch [x; x] with the contexts
    [uncond; cond] -> (e_u, e_c); fp32, unmixed (ddim.py:150-158)."""
    if not pair:
        return None, model(sd, x, t, conds, ratios, c_types=c_types, **kw)
    c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
    e_u, e_c = model(sd, torch.cat([x] * 2), torch.cat([t] * 2), c_in, ratios, c_types=c_types, **kw).chunk(2)
    return e_u, e_c


def p_sample_ddim(sd, x, conds, unconds, t, index, sched, scale, c_types=("text",), ratios=None, noise=None, temperature=1.0,
                  **kw):
    """DDIMSampler.p_sample_ddim / _multicontext, ddim.py:129-171, 244-298.  noise: the step's standard normal z (shaped like
    x), which adds sigma_t * temperature * z; None leaves the term out (eta = 0)."""
    b = x.shape[0]
    e_u, e_c = cfg_pass(apply_model, sd, x, t, conds, unconds, scale != 1.0, ratios, c_types, **kw)
    e_t = e_c if e_u is None else e_u + scale * (e_c - e_u)
    shape = [b, 1, 1, 1]
    a_t = torch.full(shape, float(sched["alphas"][index]))
    a_prev = torch.full(shape, float(sched["alphas_prev"][index]))
    sigma_t = torch.full(shape, float(sched["sigmas"][index]))
    s1m = torch.full(shape, float(sched["sqrt_one_minus_alphas"][index]))
    pred_x0 = (x - s1m * e_t) / a_t.sqrt()
    dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t
    x_prev = a_prev.sqrt() * pred_x0 + dir_xt
    if noise is not None:
        x_prev = x_prev + sigma_t * temperature * noise
    return x_prev, pred_x0, e_t


def ddim_sample_text(sd, x_T, conds, unconds, steps, scale=7.5, c_types=("text",), num_ddpm=1000, **kw):
    """DDIMSampler.sample (ddim.py:58-171) on a [n, 768] text latent: the same loop as ddim_sample with apply_model_text inside
    (app.py:384-434: inference_i2t / inference_t2t before the Optimus decode).  eta = 0."""
    sched = ddim_schedule(ddpm_schedule(num_ddpm)["alphas_cumprod"], steps)
    x = x_T
    b = x.shape[0]
    for i in range(steps):
        index = steps - i - 1
        t = torch.full((b,), int(sched["timesteps"][index]), dtype=torch.long)
        e_u, e_c = cfg_pass(apply_model_text, sd, x, t, conds, unconds, True, c_types=c_types, **kw)
        e_t = e_u + scale * (e_c - e_u)
        a_t, a_prev = float(sched["alphas"][index]), float(sched["alphas_prev"][index])
        s1m = float(sched["sqrt_one_minus_alphas"][index])
        pred_x0 = (x - s1m * e_t) / a_t ** 0.5
        x = a_prev ** 0.5 * pred_x0 + (1.0 - a_prev) ** 0.5 * e_t
    return x


def q_sample(x_start, t, noise, num_ddpm=1000):
    """VD_v2_0.q_sample, vd.py:221-224: sqrt(ac_t) * x0 + sqrt(1 - ac_t) * noise (per-row t)."""
    sch = ddpm_schedule(num_ddpm)     # sqrt taken in fp64, stored fp32 — as the reference's registered buffers
    shape = (-1,) + (1,) * (x_start.dim() - 1)
    return (sch["sqrt_alphas_cumprod"][t].reshape(shape) * x_start +
            sch["sqrt_one_minus_alphas_cumprod"][t].reshape(shape) * noise)


def img2img_start(x0, noise, timesteps, k, num_ddpm=1000):
    """The img2img start, ddim.py:97-103: (x0 noised to timesteps[k] with q_sample, the first k timesteps to walk)."""
    t0 = torch.full((x0.shape[0],), int(timesteps[k]), dtype=torch.long)
    return q_sample(x0, t0, noise, num_ddpm), timesteps[:k]


def ddim_sample(sd, x_T, conds, unconds, steps, scale=7.5, c_types=("text",), ratios=None, eta=0.0,
                num_ddpm=1000, collect=False, x0=None, x0_forward_timesteps=None, x0_noise=None, noise=None, temperature=1.0,
                timesteps=None, **kw):
    """DDIMSampler.sample / ddim_sampling, ddim.py:58-127 with x_T injected.  With x0 the img2img start from x0 and x0_noise
    (x_T is ignored).  eta > 0 needs noise(index) -> the step's z; timesteps: the grid (default DDIM's uniform one)."""
    assert eta == 0.0 or noise is not None
    sched = ddim_schedule(ddpm_schedule(num_ddpm)["alphas_cumprod"], steps, eta, timesteps)
    ts = sched["timesteps"]
    x = x_T
    if x0 is not None:
        x, ts = img2img_start(x0, x0_noise, ts, x0_forward_timesteps, num_ddpm)
    trace = []
    for i, step in enumerate(np.flip(ts)):
        index = len(ts) - i - 1
        t = torch.full((x.shape[0],), int(step), dtype=torch.long)
        z = None if eta == 0.0 else noise(index)
        x, pred_x0, e_t = p_sample_ddim(sd, x, conds, unconds, t, index, sched, scale, c_types, ratios, z, temperature, **kw)
        if collect:
            trace.append({"x": x.clone(), "pred_x0": pred_x0.clone(), "e_t": e_t.clone()})
    return (x, trace) if collect else x


def plms_sample(sd, x_T, conds, unconds, steps, scale=7.5, c_types=("text",), ratios=None, num_ddpm=1000, **kw):
    """PLMS (Liu et al. 2022; CompVis latent-diffusion plms.py) on the same apply_model — NOT in the reference
    (parity unpinned): Adams-Bashforth eps history, pseudo improved-Euler first step, eta = 0 DDIM update."""
    sched = ddim_schedule(ddpm_schedule(num_ddpm)["alphas_cumprod"], steps, 0.0)
    ts = sched["timesteps"]
    flip = np.flip(ts)
    b = x_T.shape[0]

    def eps(x, step):
        t = torch.full((b,), int(step), dtype=torch.long)
        e_u, e_c = cfg_pass(apply_model, sd, x, t, conds, unconds, scale != 1.0, ratios, c_types, **kw)
        return e_c if e_u is None else e_u + scale * (e_c - e_u)

    def update(x, e, index):
        a_t, a_prev, s1m = float(sched["alphas"][index]), float(sched["alphas_prev"][index]), float(sched["sqrt_one_minus_alphas"][index])
        pred_x0 = (x - s1m * e) / math.sqrt(a_t)
        return math.sqrt(a_prev) * pred_x0 + math.sqrt(1.0 - a_prev) * e

    x, old = x_T, []
    for i, step in enumerate(flip):
        index = len(ts) - i - 1
        e_t = eps(x, step)
        if len(old) == 0:
            e_p = (e_t + eps(update(x, e_t, index), flip[min(i + 1, len(ts) - 1)])) / 2
        elif len(old) == 1:
            e_p = (3 * e_t - old[-1]) / 2
        elif len(old) == 2:
            e_p = (23 * e_t - 16 * old[-1] + 5 * old[-2]) / 12
        else:
            e_p = (55 * e_t - 59 * old[-1] + 37 * old[-2] - 9 * old[-3]) / 24
        x = update(x, e_p, index)
        old.append(e_t)
        old = old[-3:]
    return x


# ------------------------------------------------------------------------------------------------
# AutoencoderKL (kl-f8)
# ------------------------------------------------------------------------------------------------
def _swish(x):
    return x * torch.sigmoid(x)


def vae_resnet(sd, p, x, rnd=None):
    """ResnetBlock.forward with temb=None, autokl_modules.py:119-141; GN eps 1e-6."""
    r = rnd or _identity
    h = r("conv1", F.conv2d(r("gn1", _swish(_gn(x, sd, p + ".norm1", 1e-6))), sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], padding=1))
    h = F.conv2d(r("gn2", _swish(_gn(h, sd, p + ".norm2", 1e-6))), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"], padding=1)
    if (p + ".nin_shortcut.weight") in sd:
        x = F.conv2d(x, sd[p + ".nin_shortcut.weight"], sd[p + ".nin_shortcut.bias"])
    return r("out", x + h)


def vae_attn(sd, p, x, rnd=None):
    """AttnBlock.forward, autokl_modules.py:178-202 (single head, d = C).  With a rounding hook, v is rounded without its bias
    and b_v is added after P v (the softmax rows sum to 1)."""
    r = rnd or _identity
    h_ = r("gn", _gn(x, sd, p + ".norm", 1e-6))
    q = r("q", F.conv2d(h_, sd[p + ".q.weight"], sd[p + ".q.bias"]))
    k = r("k", F.conv2d(h_, sd[p + ".k.weight"], sd[p + ".k.bias"]))
    b, c, h, w = q.shape
    q = q.reshape(b, c, h * w).permute(0, 2, 1)
    k = k.reshape(b, c, h * w)
    if rnd is None:
        v = F.conv2d(h_, sd[p + ".v.weight"], sd[p + ".v.bias"])
        w_ = torch.bmm(q, k) * (int(c) ** (-0.5))
        w_ = F.softmax(w_, dim=2)
        v = v.reshape(b, c, h * w)
        h_ = torch.bmm(v, w_.permute(0, 2, 1)).reshape(b, c, h, w)
    else:
        v = r("v", F.conv2d(h_, sd[p + ".v.weight"])).reshape(b, c, h * w)
        w_ = r("p", F.softmax(r("s", torch.bmm(q, k)) * (int(c) ** (-0.5)), dim=2))
        h_ = r("o", torch.bmm(v, w_.permute(0, 2, 1)) + sd[p + ".v.bias"][None, :, None]).reshape(b, c, h, w)
    return r("out", x + F.conv2d(h_, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"]))


def vae_downsample(sd, p, x):
    """Downsample with conv, autokl_modules.py:60-79: pad (0, 1, 0, 1), then conv3x3 stride 2."""
    x = F.pad(x, (0, 1, 0, 1), mode="constant", value=0)
    return F.conv2d(x, sd[p + ".conv.weight"], sd[p + ".conv.bias"], stride=2)


def vae_decode(sd, z, scale_factor=0.18215, ch_mult=(1, 2, 4, 4), num_res_blocks=2, prefix="vae.image"):
    """VD_v2_0.vae_decode (vd.py:291-298) -> AutoencoderKL.decode (autokl.py:44-49) -> Decoder.forward
    (autokl_modules.py:535-568)."""
    z = 1.0 / scale_factor * z
    z = F.conv2d(z, sd[prefix + ".post_quant_conv.weight"], sd[prefix + ".post_quant_conv.bias"])
    D = prefix + ".decoder"
    h = F.conv2d(z, sd[D + ".conv_in.weight"], sd[D + ".conv_in.bias"], padding=1)
    h = vae_resnet(sd, D + ".mid.block_1", h)
    h = vae_attn(sd, D + ".mid.attn_1", h)
    h = vae_resnet(sd, D + ".mid.block_2", h)
    for lvl in reversed(range(len(ch_mult))):
        for blk in range(num_res_blocks + 1):
            h = vae_resnet(sd, f"{D}.up.{lvl}.block.{blk}", h)
        if lvl != 0:
            h = upsample(sd, f"{D}.up.{lvl}.upsample", h)
    h = F.conv2d(_swish(_gn(h, sd, D + ".norm_out", 1e-6)), sd[D + ".conv_out.weight"], sd[D + ".conv_out.bias"], padding=1)
    return torch.clamp((h + 1) / 2, 0, 1)


def vae_encode(sd, x, noise=None, scale_factor=0.18215, ch_mult=(1, 2, 4, 4), num_res_blocks=2, prefix="vae.image"):
    """VD_v2_0.vae_encode (vd.py:282-289) -> AutoencoderKL.encode (autokl.py:30-42) -> Encoder.forward
    (autokl_modules.py:434-459) -> DiagonalGaussianDistribution.sample (distributions.py:24-37) with the
    standard-normal draw injected (`noise`; None = posterior mean)."""
    x = x * 2 - 1
    E = prefix + ".encoder"
    h = F.conv2d(x, sd[E + ".conv_in.weight"], sd[E + ".conv_in.bias"], padding=1)
    for lvl in range(len(ch_mult)):
        for blk in range(num_res_blocks):
            h = vae_resnet(sd, f"{E}.down.{lvl}.block.{blk}", h)
        if lvl != len(ch_mult) - 1:
            h = vae_downsample(sd, f"{E}.down.{lvl}.downsample", h)
    h = vae_resnet(sd, E + ".mid.block_1", h)
    h = vae_attn(sd, E + ".mid.attn_1", h)
    h = vae_resnet(sd, E + ".mid.block_2", h)
    h = F.conv2d(_swish(_gn(h, sd, E + ".norm_out", 1e-6)), sd[E + ".conv_out.weight"], sd[E + ".conv_out.bias"], padding=1)
    moments = F.conv2d(h, sd[prefix + ".quant_conv.weight"], sd[prefix + ".quant_conv.bias"])
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    z = mean if noise is None else mean + torch.exp(0.5 * logvar) * noise
    return scale_factor * z


# ------------------------------------------------------------------------------------------------
# CLIP ViT-L/14 context encoders (third-party arithmetic restated; see module docstring)
# ------------------------------------------------------------------------------------------------
def _clip_layer(sd, p, x, heads, mask):
    """One HF CLIPEncoderLayer: pre-LN MHA (scale on q) + pre-LN MLP with quick_gelu."""
    b, n, c = x.shape
    d = c // heads
    h = F.layer_norm(x, (c,), sd[p + ".layer_norm1.weight"], sd[p + ".layer_norm1.bias"], 1e-5)
    proj = lambda name: F.linear(h, sd[f"{p}.self_attn.{name}.weight"], sd[f"{p}.self_attn.{name}.bias"])
    split = lambda t: t.view(b, n, heads, d).permute(0, 2, 1, 3)
    q, k, v = split(proj("q_proj")), split(proj("k_proj")), split(proj("v_proj"))
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * d ** -0.5
    if mask is not None:
        sim = sim + mask
    o = torch.einsum("bhij,bhjd->bhid", sim.softmax(-1), v).permute(0, 2, 1, 3).reshape(b, n, c)
    x = x + F.linear(o, sd[p + ".self_attn.out_proj.weight"], sd[p + ".self_attn.out_proj.bias"])
    h = F.layer_norm(x, (c,), sd[p + ".layer_norm2.weight"], sd[p + ".layer_norm2.bias"], 1e-5)
    h = F.linear(h, sd[p + ".mlp.fc1.weight"], sd[p + ".mlp.fc1.bias"])
    h = h * torch.sigmoid(1.702 * h)
    return x + F.linear(h, sd[p + ".mlp.fc2.weight"], sd[p + ".mlp.fc2.bias"])


def clip_text_encode(sd, tokens, heads=12, layers=12, prefix="ctx.text.model"):
    """CLIPTextContextEncoder.encode after tokenisation, clip.py:57-62: text_model -> text_projection on
    all tokens -> divide by || text_projection(pooled) ||, pooled = hidden state at argmax(token id)
    (the EOS token, id 49407, is the largest id)."""
    T = prefix + ".text_model"
    b, n = tokens.shape
    x = sd[T + ".embeddings.token_embedding.weight"][tokens] + sd[T + ".embeddings.position_embedding.weight"][:n]
    mask = torch.full((n, n), float("-inf")).triu(1)
    for i in range(layers):
        x = _clip_layer(sd, f"{T}.encoder.layers.{i}", x, heads, mask)
    c = x.shape[-1]
    x = F.layer_norm(x, (c,), sd[T + ".final_layer_norm.weight"], sd[T + ".final_layer_norm.bias"], 1e-5)
    pooled = x[torch.arange(b), tokens.argmax(dim=-1)]
    z = F.linear(x, sd[prefix + ".text_projection.weight"])
    zp = F.linear(pooled, sd[prefix + ".text_projection.weight"])
    return z / torch.norm(zp.unsqueeze(1), dim=-1, keepdim=True)


def clip_image_encode_wmask(sd, pixels, masks, heads=16, layers=24, patch=14, prefix="ctx.image.model"):
    """CLIPImageContextEncoder._encode_wmask, clip.py:103-143: masks [b,1,h,w] -> clamp, bilinear resize to 224x224; an all-ones
    mask is the unmasked encode (:110-111); otherwise every token embedding (class token: the mask's global mean, patch tokens:
    the mean of the mask over the patch = conv with a ones kernel / P^2, :114-121) is scaled AFTER the position embedding and
    BEFORE pre_layrnorm (:124-133), and the normalised output is scaled by the same factors again (:141).
    Parity note: the reference's own masked path cannot run on transformers 5.5.0 (its patched embeddings.forward lacks the
    `interpolate_pos_encoding` keyword), so this restatement is pinned to the reference's LINES, not to its output."""
    masks = F.interpolate(torch.clamp(masks, 0, 1).float(), [224, 224], mode="bilinear")
    if masks.sum() == masks.numel():
        return clip_image_encode(sd, pixels, heads, layers, patch, prefix)
    gscale = masks.mean(dim=[1, 2, 3], keepdim=True).flatten(2)
    vtoken = F.conv2d(masks, torch.ones(1, 1, patch, patch), stride=patch).flatten(2).transpose(1, 2) / float(patch * patch)
    vtoken_mask = torch.cat([gscale, vtoken], dim=1)                      # [b, 257, 1]
    return clip_image_encode(sd, pixels, heads, layers, patch, prefix, tok_scale=vtoken_mask) * vtoken_mask


def clip_image_encode(sd, pixels, heads=16, layers=24, patch=14, prefix="ctx.image.model", tok_scale=None):
    """CLIPImageContextEncoder._encode after the CLIPProcessor, clip.py:95-101: vision_model ->
    post_layernorm on ALL tokens of last_hidden_state -> visual_projection -> divide by ||token 0||.
    pixels: [b,3,224,224] already resized/normalised."""
    V = prefix + ".vision_model"
    b = pixels.shape[0]
    pe = F.conv2d(pixels, sd[V + ".embeddings.patch_embedding.weight"], stride=patch).flatten(2).transpose(1, 2)
    cls = sd[V + ".embeddings.class_embedding"].expand(b, 1, -1)
    x = torch.cat([cls, pe], dim=1) + sd[V + ".embeddings.position_embedding.weight"][None]
    if tok_scale is not None:           # masked variant (clip.py:124-133)
        x = x * tok_scale
    c = x.shape[-1]
    x = F.layer_norm(x, (c,), sd[V + ".pre_layrnorm.weight"], sd[V + ".pre_layrnorm.bias"], 1e-5)
    for i in range(layers):
        x = _clip_layer(sd, f"{V}.encoder.layers.{i}", x, heads, None)
    # HF returns last_hidden_state WITHOUT post_layernorm (only the pooled token gets it); the reference
    # then applies post_layernorm to every token itself (clip.py:97-98)
    z = F.layer_norm(x, (c,), sd[V + ".post_layernorm.weight"], sd[V + ".post_layernorm.bias"], 1e-5)
    z = F.linear(z, sd[prefix + ".visual_projection.weight"])
    return z / torch.norm(z[:, 0:1], dim=-1, keepdim=True)
