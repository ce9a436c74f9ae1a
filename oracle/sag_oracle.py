"""Self-attention guidance oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

Restates lib/model_zoo/sag.py from its specification: vd_oracle.apply_model (the fp32 UNet) with a hook on the mid block's
self-attention (the 'ctx' of the layout between the last 'save' and the first 'load', found from the layout, never from the token
count), the key mass and its mask, the reflect-padded 9 x 9 Gaussian blur as one 2-D depthwise conv2d, nearest upsampling, the
re-noise, the second pass on the uncond (CFG) or cond contexts and the guide, all in fp64 on the UNet's fp32 outputs.  The walk is
DDIM (DPM-Solver++ of order 1, equal to DDIM at eta 0) or DPM-Solver++ 2M through dpm_solver_oracle.walk, with inpaint_oracle's
blend as its `after` under a mask.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import dpm_sde_oracle as G
from . import inpaint_oracle as I
from . import panorama_oracle as P
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
    """The guided eps at timestep t of x [bs, C, H, W] (fp64 -> fp32 UNet input), fp64.  masses, when a list, receives the mass:
    [bs, N] fp64, sum_i r_i (1/H) sum_h sum_p P_i[b, h, p, j] of the mid block's self-attention over the first pass's first bs
    rows (the uncond rows under CFG), r_i the normalised ratio of context i."""
    bs = x.shape[0]
    cfg = scale != 1.0
    tt = torch.full((bs,), int(t), dtype=torch.long)
    mid, _ = mid_block(O.unet_layout())
    r = O.context_weights(ratios, len(conds))
    mass = [None]

    def hook_for(j, idx):
        def hook(probs, cross):
            if not cross:
                m = r[j] * probs[:bs].double().sum(dim=2).mean(dim=1)
                mass[0] = m if mass[0] is None else mass[0] + m
            return probs
        return hook if idx == mid else None

    e_u, e_c = O.cfg_pass(O.apply_model, sd, x.float(), tt, conds, unconds, cfg, ratios, c_types, hook_for=hook_for, **kw)
    e_u, e_c = None if e_u is None else e_u.double(), e_c.double()
    e_src = e_u if cfg else e_c
    if masses is not None:
        masses.append(mass[0])
    x_deg = degrade(x.double(), e_src, mass[0], a)
    e_deg = O.apply_model(sd, x_deg.float(), tt, unconds if cfg else conds, ratios, c_types=c_types, **kw).double()
    d = s * (e_src - e_deg)
    return (e_u + d) + scale * (e_c - e_u) if cfg else e_c + d


def sample(sd, x_T, conds, unconds, steps, s, sampler="ddim", scale=7.5, c_types=("text",), ratios=None, x0=None, mask=None,
           noise_fn=None, masses=None, num_ddpm=1000, order=2, grid_name="uniform", eta=0.0, noise=None, **kw):
    """The SAG walk from x_T [bs, C, H, W]: DDIM (order 1 at eta 0, the stochastic DDIM step at eta > 0) or DPM-Solver++ of
    `order` in fp64, with the inpainting blend when mask (latent [bs or 1, 1, H, W]) and x0 are given (noise_fn(i) -> z_i, the
    full walk's masked start).  grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature)."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    ts = sched["timesteps"]
    acn = ac.numpy()
    order = 1 if sampler == "ddim" else order

    def eps_fn(xv, i):
        a = float(np.float64(acn[ts[i]]))
        return sag_eps(sd, torch.from_numpy(np.asarray(xv)), ts[i], conds, unconds, scale, s, a, c_types, ratios, masses,
                       **kw).numpy()

    x, after = x_T, None
    if mask is not None:
        x = I.start(x_T.float(), x0.float(), mask.float(), acn, int(ts[-1]))
        after = I.blend_after(acn, ts, x0, mask, noise_fn)
    if sampler == "ddim" and eta != 0:
        x = x.double().numpy()
        for i in range(len(ts) - 1, -1, -1):
            x = P.ddim_update(x, eps_fn(x, i), float(sched["alphas"][i]), float(sched["alphas_prev"][i]), float(sched["sigmas"][i]),
                              np.asarray(noise(i), dtype=np.float64))
            x = x if after is None else after(i, x)
        return torch.from_numpy(x).float()
    out = G.dpm_walk(x.double().numpy(), eps_fn, acn, ts, order, eta, noise, after=after)
    return torch.from_numpy(out).float()
