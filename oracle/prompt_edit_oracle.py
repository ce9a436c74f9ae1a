"""Prompt-to-Prompt oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

Restates lib/model_zoo/prompt_edit.py as P2P computes it: on materialised attention probabilities of the fp32 UNet of
vd_oracle (its pieces, with an attention hook on the text context's SpatialTransformers), with the mapper einsum, the equalizer
product, the alpha mix, the self-map replacement, and LocalBlend with max_pool2d / nearest interpolate.  It never forms the
factored A * ctx contexts, so comparing against it checks the factoring too.  The walk is DDIM or DPM-Solver++ in fp64.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import dpm_solver_oracle as D
from . import vd_oracle as O


def _attention(sd, p, x, context, heads, hook):
    """vd_oracle.cross_attention with hook(probs [b, h, n, L], is_cross) -> the probabilities that weight V."""
    cross = context is not None
    context = x if context is None else context
    q = F.linear(x, sd[p + ".to_q.weight"])
    k = F.linear(context, sd[p + ".to_k.weight"])
    v = F.linear(context, sd[p + ".to_v.weight"])
    b, n, c = q.shape
    d = c // heads
    split = lambda t: t.view(b, t.shape[1], heads, d).permute(0, 2, 1, 3)
    q, k, v = split(q), split(k), split(v)
    probs = (torch.einsum("bhid,bhjd->bhij", q, k) * d ** -0.5).softmax(dim=-1)
    if hook is not None:
        probs = hook(probs, cross)
    out = torch.einsum("bhij,bhjd->bhid", probs, v).permute(0, 2, 1, 3).reshape(b, n, c)
    return F.linear(out, sd[p + ".to_out.0.weight"], sd[p + ".to_out.0.bias"])


def _spatial_transformer(sd, p, x, context, heads, hook):
    b, c, h, w = x.shape
    x_in = x
    x = O._gn(x, sd, p + ".norm", 1e-6)
    x = F.conv2d(x, sd[p + ".proj_in.weight"], sd[p + ".proj_in.bias"])
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, c)
    t = p + ".transformer_blocks.0"
    ln = lambda y, nm: F.layer_norm(y, (c,), sd[f"{t}.{nm}.weight"], sd[f"{t}.{nm}.bias"], 1e-5)
    x = _attention(sd, t + ".attn1", ln(x, "norm1"), None, heads, hook) + x
    x = _attention(sd, t + ".attn2", ln(x, "norm2"), context, heads, hook) + x
    hdn = F.linear(ln(x, "norm3"), sd[t + ".ff.net.0.proj.weight"], sd[t + ".ff.net.0.proj.bias"])
    val, gate = hdn.chunk(2, dim=-1)
    x = F.linear(val * F.gelu(gate), sd[t + ".ff.net.2.weight"], sd[t + ".ff.net.2.bias"]) + x
    x = x.reshape(b, h, w, c).permute(0, 3, 1, 2)
    return F.conv2d(x, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"]) + x_in


def apply_model(sd, x, timesteps, contexts, ratios, c_types, hook, model_channels=320, num_heads=8):
    """vd_oracle.apply_model (image latents) with `hook` on the SpatialTransformers of the text context."""
    layout = O.unet_layout(model_channels=model_channels, num_heads=num_heads)
    Dp = "diffuser.image"
    t_emb = O.timestep_embedding(timesteps, model_channels)
    emb = F.linear(F.silu(F.linear(t_emb, sd[Dp + ".time_embed.0.weight"], sd[Dp + ".time_embed.0.bias"])),
                   sd[Dp + ".time_embed.2.weight"], sd[Dp + ".time_embed.2.bias"])
    r = np.array(ratios if ratios is not None else [1.0] * len(contexts), dtype=np.float64)
    r = r / r.sum()
    hs, h = [], x
    for kind, idx, _ in layout:
        if kind == "conv_in":
            h = F.conv2d(h, sd[f"{Dp}.data_blocks.{idx}.0.weight"], sd[f"{Dp}.data_blocks.{idx}.0.bias"], padding=1)
        elif kind == "res":
            h = O.resblock(sd, f"{Dp}.data_blocks.{idx}.0", h, emb)
        elif kind == "down":
            h = F.conv2d(h, sd[f"{Dp}.data_blocks.{idx}.0.op.weight"], sd[f"{Dp}.data_blocks.{idx}.0.op.bias"], stride=2, padding=1)
        elif kind == "up":
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = F.conv2d(h, sd[f"{Dp}.data_blocks.{idx}.0.conv.weight"], sd[f"{Dp}.data_blocks.{idx}.0.conv.bias"], padding=1)
        elif kind == "out":
            p = f"{Dp}.data_blocks.{idx}.0"
            h = F.conv2d(F.silu(O._gn(h, sd, p + ".0", 1e-5)), sd[p + ".2.weight"], sd[p + ".2.bias"], padding=1)
        elif kind == "ctx":
            terms = [_spatial_transformer(sd, f"diffuser.{ct}.context_blocks.{idx}.0", h, c, num_heads,
                                          hook if ct == "text" else None) for ct, c in zip(c_types, contexts)]
            h = terms[0] if len(terms) == 1 else sum(t * ri for t, ri in zip(terms, r))
        elif kind == "save":
            hs.append(h)
        elif kind == "load":
            h = torch.cat([h, hs.pop()], dim=1)
    return h


class P2P(object):
    """The P2P controller over the CFG batch [uncond; cond] of n prompts.  kind 'replace' (M [n-1, L, L]), 'refine'
    (mp [n-1, L], alpha [n-1, L]) or 'reweight'; c [n-1, L] the equalizer; w [n, L] blend words or None."""

    def __init__(self, n, kind, T, cross_steps, self_steps, c, H, W, M=None, mp=None, alpha=None, w=None, threshold=0.3,
                 blend_start=0.0, cfg=True):
        self.n, self.kind, self.T, self.c, self.M, self.mp, self.alpha, self.w = n, kind, T, c, M, mp, alpha, w
        self.tc, self.ts = math.floor(cross_steps * T), math.floor(self_steps * T)
        self.tb, self.threshold, self.cfg = math.floor(blend_start * T), threshold, cfg
        self.h4, self.w4 = ((H + 1) // 2 + 1) // 2, ((W + 1) // 2 + 1) // 2
        self.i = 0
        self.maps = torch.zeros(n, self.h4 * self.w4, dtype=torch.float64)

    def hook(self, probs, cross):
        n = self.n
        c0 = n if self.cfg else 0
        N = probs.shape[2]
        cond = probs[c0:c0 + n]
        out = probs.clone()
        if cross:
            if self.w is not None and N == self.h4 * self.w4:      # the row's own probabilities, before the edit
                w = torch.as_tensor(self.w, dtype=torch.float64)
                self.maps += (cond.double() * w[:, None, None, :]).sum(dim=(1, 3))
            if self.i < self.tc:
                base = cond[0]
                for t in range(1, n):
                    c = torch.as_tensor(self.c[t - 1], dtype=probs.dtype)
                    if self.kind == "replace":
                        e = torch.einsum("hpw,wn->hpn", base, torch.as_tensor(self.M[t - 1], dtype=probs.dtype))
                    elif self.kind == "refine":
                        a = torch.as_tensor(self.alpha[t - 1], dtype=probs.dtype)
                        e = base[:, :, torch.as_tensor(self.mp[t - 1])] * a + cond[t] * (1 - a)
                    else:
                        e = base
                    out[c0 + t] = e * c
        elif N <= self.h4 * self.w4 and self.i < self.ts:
            for t in range(1, n):
                out[c0 + t] = cond[0]
        return out

    def blend(self, x):
        """LocalBlend after step i on x [n, C, H, W] (fp64)."""
        if self.w is None or self.i < self.tb:
            return x
        m = self.maps.view(self.n, 1, self.h4, self.w4)
        m = F.max_pool2d(m, (3, 3), (1, 1), padding=(1, 1))
        m = F.interpolate(m, size=x.shape[2:])
        mx = m.amax(dim=(2, 3), keepdim=True)
        m = torch.where(mx > 0, m / torch.where(mx > 0, mx, torch.ones_like(mx)), torch.zeros_like(m)).gt(self.threshold)
        m = m[:1] | m[1:]
        out = x.clone()
        out[1:] = torch.where(m, x[1:], x[:1])
        return out


def _eps_fn(sd, ctl, conds, unconds, scale, c_types, ratios, kw):
    def eps(x, t):
        tt = torch.full((x.shape[0],), int(t), dtype=torch.long)
        xf = x.float()
        c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
        e_u, e_c = apply_model(sd, torch.cat([xf] * 2), torch.cat([tt] * 2), c_in, ratios, c_types, ctl.hook, **kw).chunk(2)
        return e_u.double() + scale * (e_c.double() - e_u.double())
    return eps


def sample(sd, ctl, x_T, conds, unconds, steps, sampler="ddim", order=2, scale=7.5, c_types=("text",), ratios=None,
           num_ddpm=1000, **kw):
    """The edited walk from x_T [n, C, H, W] (fp64 state, fp32 UNet) with the local blend after every step."""
    ac = O.ddpm_schedule(num_ddpm)["alphas_cumprod"]
    sched = O.ddim_schedule(ac, steps)
    ts = sched["timesteps"]
    eps = _eps_fn(sd, ctl, conds, unconds, scale, c_types, ratios, kw)
    x = x_T.double()
    if sampler == "ddim":
        for k, i in enumerate(range(steps - 1, -1, -1)):
            ctl.i = k
            a, ap = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
            e = eps(x, ts[i])
            x = np.sqrt(ap) * (x - np.sqrt(1.0 - a) * e) / np.sqrt(a) + np.sqrt(1.0 - ap) * e
            x = ctl.blend(x)
        return x
    alpha, sigma, lam, alpha_to, sigma_to = (np.asarray(a, dtype=np.float64).tolist() for a in D.coefficients(ac.numpy(), ts))
    x0s, lams = [], []
    for k, i in enumerate(range(steps - 1, -1, -1)):
        ctl.i = k
        xp = (x - sigma[i] * eps(x, ts[i])) / alpha[i]
        h = math.log(alpha_to[i]) - math.log(sigma_to[i]) - lam[i]
        phi1 = math.expm1(-h)
        o = D.step_order(order, k, i, steps)
        xn = sigma_to[i] / sigma[i] * x - alpha_to[i] * phi1 * xp
        if o == 2:
            r0 = (lam[i] - lams[-1]) / h
            xn = xn - 0.5 * alpha_to[i] * phi1 * (xp - x0s[-1]) / r0
        elif o == 3:
            raise NotImplementedError("order 3 is not restated here")
        x = ctl.blend(xn)
        x0s.append(xp)
        lams.append(lam[i])
    return x
