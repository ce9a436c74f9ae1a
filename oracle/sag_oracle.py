"""Self-attention guidance oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

Restates lib/model_zoo/sag.py from its specification: the fp32 UNet of vd_oracle's pieces with a hook on the mid block's
self-attention (the 'ctx' of the layout between the last 'save' and the first 'load', found from the layout, never from the token
count), the key mass and its mask, the reflect-padded 9 x 9 Gaussian blur as one 2-D depthwise conv2d, nearest upsampling, the
re-noise, the second pass on the uncond (CFG) or cond contexts and the guide, all in fp64 on the UNet's fp32 outputs.  The walk is
DDIM (DPM-Solver++ of order 1, equal to DDIM at eta 0) or DPM-Solver++ 2M through dpm_solver_oracle, or the masked walk of
inpaint_oracle.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import dpm_solver_oracle as D
from . import inpaint_oracle as I
from . import prompt_edit_oracle as P
from . import vd_oracle as O


def taps():
    """The 1-D Gaussian of sigma 1 on k = -4 .. 4, normalised to sum 1 (fp64)."""
    k = np.arange(-4, 5, dtype=np.float64)
    g = np.exp(-0.5 * k * k)
    return g / g.sum()


def blur(x):
    """x [n, C, H, W] fp64 -> the depthwise 9 x 9 Gaussian (outer product of taps()) with reflect padding by 4."""
    g = torch.from_numpy(taps())
    k2 = torch.outer(g, g).to(x.dtype)
    C = x.shape[1]
    return F.conv2d(F.pad(x, (4, 4, 4, 4), mode="reflect"), k2.expand(C, 1, 9, 9).contiguous(), groups=C)


def nearest_index(n_out, n_in):
    """the source row of each of n_out rows upsampled from n_in by nearest neighbour: floor(y n_in / n_out), in integers"""
    return (np.arange(n_out) * n_in) // n_out


def mid_block(layout):
    """(index of the mid block's context block, number of stride-2 downsamples before it) in a vd_oracle.unet_layout"""
    first_load = next(n for n, (kind, _, _) in enumerate(layout) if kind == "load")
    n_mid = max(n for n, (kind, _, _) in enumerate(layout[:first_load]) if kind == "ctx")
    return layout[n_mid][1], sum(1 for kind, _, _ in layout[:n_mid] if kind == "down")


def mid_size(H, W, layout=None):
    """the mid block's token grid: each stride-2 conv (kernel 3, padding 1) maps n to floor((n - 1) / 2) + 1"""
    _, downs = mid_block(layout or O.unet_layout())
    for _ in range(downs):
        H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    return H, W


def apply_model(sd, x, timesteps, contexts, ratios, c_types, rows=None, model_channels=320, num_heads=8):
    """vd_oracle.apply_model (image latents) -> (eps, mass): mass [len(rows), N] fp64, sum_i r_i (1/H) sum_h sum_p P_i[b, h, p, j]
    of the mid block's self-attention over batch rows `rows` (None: no mass)."""
    layout = O.unet_layout(model_channels=model_channels, num_heads=num_heads)
    mid, _ = mid_block(layout)
    Dp = "diffuser.image"
    t_emb = O.timestep_embedding(timesteps, model_channels)
    emb = F.linear(F.silu(F.linear(t_emb, sd[Dp + ".time_embed.0.weight"], sd[Dp + ".time_embed.0.bias"])),
                   sd[Dp + ".time_embed.2.weight"], sd[Dp + ".time_embed.2.bias"])
    r = np.array(ratios if ratios is not None else [1.0] * len(contexts), dtype=np.float64)
    r = r / r.sum()
    mass = [None]

    def hook_for(ri):
        def hook(probs, cross):
            if not cross:
                m = ri * probs[rows].double().sum(dim=2).mean(dim=1)
                mass[0] = m if mass[0] is None else mass[0] + m
            return probs
        return hook

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
            terms = [P._spatial_transformer(sd, f"diffuser.{ct}.context_blocks.{idx}.0", h, c, num_heads,
                                            hook_for(ri) if idx == mid and rows is not None else None)
                     for ct, c, ri in zip(c_types, contexts, r)]
            h = terms[0] if len(terms) == 1 else sum(t * ri for t, ri in zip(terms, r))
        elif kind == "save":
            hs.append(h)
        elif kind == "load":
            h = torch.cat([h, hs.pop()], dim=1)
    return h, mass[0]


def degrade(x, e, mass, a):
    """x, e fp64 [bs, C, H, W]; mass [bs, hm * wm]; a = a_t -> x_deg"""
    bs, _, H, W = x.shape
    hm, wm = mid_size(H, W)
    M = (mass > 1.0).double().view(bs, 1, hm, wm)
    M = M[:, :, nearest_index(H, hm)][:, :, :, nearest_index(W, wm)]
    x0 = (x - np.sqrt(1.0 - a) * e) / np.sqrt(a)
    x0d = M * blur(x0) + (1 - M) * x0
    return np.sqrt(a) * x0d + np.sqrt(1.0 - a) * e


def sag_eps(sd, x, t, conds, unconds, scale, s, a, c_types=("text",), ratios=None, masses=None, **kw):
    """The guided eps at timestep t of x [bs, C, H, W] (fp64 -> fp32 UNet input), fp64.  masses, when a list, receives the mass."""
    bs = x.shape[0]
    xf = x.float()
    cfg = scale != 1.0
    tt = torch.full((bs,), int(t), dtype=torch.long)
    if cfg:
        c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
        e, mass = apply_model(sd, torch.cat([xf] * 2), torch.cat([tt] * 2), c_in, ratios, c_types, rows=slice(0, bs), **kw)
        e_u, e_c = e.double().chunk(2)
        e_src = e_u
    else:
        e, mass = apply_model(sd, xf, tt, conds, ratios, c_types, rows=slice(0, bs), **kw)
        e_u, e_c = None, e.double()
        e_src = e_c
    if masses is not None:
        masses.append(mass)
    x_deg = degrade(x.double(), e_src, mass, a)
    e_deg = apply_model(sd, x_deg.float(), tt, unconds if cfg else conds, ratios, c_types, **kw)[0].double()
    d = s * (e_src - e_deg)
    return (e_u + d) + scale * (e_c - e_u) if cfg else e_c + d


def sample(sd, x_T, conds, unconds, steps, s, sampler="ddim", scale=7.5, c_types=("text",), ratios=None, x0=None, mask=None,
           noise_fn=None, masses=None, num_ddpm=1000, **kw):
    """The SAG walk from x_T [bs, C, H, W]: DDIM (order 1) or DPM-Solver++ 2M in fp64, with the inpainting blend when mask (latent
    [bs or 1, 1, H, W]) and x0 are given (noise_fn(i) -> z_i, the full walk's masked start)."""
    ac = O.ddpm_schedule(num_ddpm)["alphas_cumprod"]
    ts = O.make_ddim_timesteps(steps, num_ddpm)
    acn = ac.numpy()
    order = 1 if sampler == "ddim" else 2

    def eps_fn(xv, i):
        a = float(np.float64(acn[ts[i]]))
        return sag_eps(sd, torch.from_numpy(np.asarray(xv)), ts[i], conds, unconds, scale, s, a, c_types, ratios, masses,
                       **kw).numpy()

    if mask is None:
        out = D.walk(x_T.double().numpy(), eps_fn, acn, ts, order)
    else:
        x = I.start(x_T.float(), x0.float(), mask.float(), acn, int(ts[-1])).double()
        out = I.dpm_walk(x.numpy(), eps_fn, acn, ts, order, x0.double().numpy(), mask.double().numpy(),
                         lambda i: noise_fn(i).double().numpy())
    return torch.from_numpy(out).float()
