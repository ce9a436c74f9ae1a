"""Region-prompt oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

A CPU restatement of the region walk of lib/model_zoo/regions.py in the paper's form (Bar-Tal et al. 2023, section 4.2), in fp64:
every step crops each window of every region's input (the canvas, or under bootstrapping m_r x + (1 - m_r)(a bg + b z) for region
r >= 1), runs one guided DDIM step per (window, region) with the region's own unconditional and conditional rows, and takes the
per-element sum of m_r x_{t-1} over windows and regions divided by n D, with m_0 = max(0, 1 - S) and D = m_0 + S.  DPM-Solver++ is
multistep, so its paper form has no per-view state; it is the canvas walk of dpm_solver_oracle.walk (with inpaint_oracle's blend
as its `after` under an inpainting mask) with the mask-weighted average of the views' guided eps.  The product averages eps in
every case; the CPU tests check that the paper-form DDIM step equals the eps average for binary masks, and that all-zero masks
reduce to the plain (windowed) walk.
"""
import numpy as np
import torch

from . import dpm_sde_oracle as G
from . import inpaint_oracle as I
from . import panorama_oracle as P
from . import vd_oracle as O


def weights(masks):
    """masks fp64 [R, bs, H, W] -> (m [R + 1, bs, H, W] with m_0 = max(0, 1 - S) first, D = m_0 + S)"""
    masks = np.asarray(masks, dtype=np.float64)
    S = masks.sum(0)
    m0 = np.maximum(0.0, 1.0 - S)
    return np.concatenate([m0[None], masks]), m0 + S


def region_inputs(x, masks, boot=None):
    """[x_0, ..., x_R]: the canvas x [bs, C, H, W] for every region, or, with boot = (bgs [R, bs, C], z [bs, C, H, W], a, b), the
    bootstrapped input m_r x + (1 - m_r)(a bg_r + b z) for r >= 1"""
    xs = [x]
    for r in range(masks.shape[0]):
        if boot is None:
            xs.append(x)
            continue
        bgs, z, a, b = boot
        m = masks[r][:, None]
        xs.append(m * x + (1.0 - m) * (a * bgs[r][:, :, None, None] + b * z))
    return xs


def _weighted_sum(x, parts_fn, masks, wins, h, w):
    """sum over windows g and regions r of m_r * parts_fn(g, r) placed on the canvas, over n D"""
    m, Dn = weights(masks)
    acc = np.zeros(x.shape, dtype=np.float64)
    cnt = np.zeros(x.shape[-2:], dtype=np.float64)
    W = x.shape[-1]
    for g, (oy, ox) in enumerate(wins):
        cols = (ox + np.arange(w)) % W
        for r in range(m.shape[0]):
            acc[..., oy:oy + h, cols] += P.crop(m[r], oy, ox, h, w)[:, None] * np.asarray(parts_fn(g, r), dtype=np.float64)
        cnt[oy:oy + h, cols] += 1
    return acc / (cnt * Dn)[:, None]


def paper_step(x, eps_fn, masks, wins, h, w, a_t, a_prev, boot=None):
    """The paper's step: one DDIM step per window crop of every region's input, mask-weighted.  eps_fn(crop, g, r) -> the guided
    eps of region r's view g."""
    xs = region_inputs(x, masks, boot)

    def part(g, r):
        xc = P.crop(xs[r], *wins[g], h, w)
        return P.ddim_update(xc, eps_fn(xc, g, r), a_t, a_prev)
    return _weighted_sum(x, part, masks, wins, h, w)


def eps_average(x, eps_fn, masks, wins, h, w, boot=None):
    """The product's form: the mask-weighted average of the views' guided eps."""
    xs = region_inputs(x, masks, boot)
    return _weighted_sum(x, lambda g, r: eps_fn(P.crop(xs[r], *wins[g], h, w), g, r), masks, wins, h, w)


def _views_eps(sd, xs, t, conds, unconds, region_conds, wins, h, w, scale, c_types, ratios, kw):
    """{(g, r): guided eps} of every view through the UNet restatement; region r's views are one batch, with its own u rows"""
    out = {}
    n, bs = len(wins), xs[0].shape[0]
    rep = lambda cs: [c.repeat(n, 1, 1) for c in cs]
    for r, xr in enumerate(xs):
        xc = torch.cat([torch.from_numpy(P.crop(xr, oy, ox, h, w).copy()).float() for oy, ox in wins])     # row g*bs + b
        tt = torch.full((n * bs,), int(t), dtype=torch.long)
        cs = conds if r == 0 else region_conds[r - 1]
        e_u, e_c = O.cfg_pass(O.apply_model, sd, xc, tt, rep(cs), rep(unconds), scale != 1.0, ratios, c_types, **kw)
        e = e_c if e_u is None else e_u + scale * (e_c - e_u)
        e = e.double().numpy().reshape(n, bs, *e.shape[1:])
        for g in range(n):
            out[g, r] = e[g]
    return out


def sample(sd, x_T, conds, unconds, region_conds, masks, steps, size=None, stride=8, circular=False, sampler="ddim", order=2,
           scale=7.5, c_types=("text",), ratios=None, bootstrap_steps=0, backgrounds=None, pick_fn=None, z_fn=None, x0=None,
           mask=None, noise_fn=None, num_ddpm=1000, grid_name="uniform", eta=0.0, noise=None, **kw):
    """The region DDIMSampler / DPMSolverSampler walk on the UNet restatement, from x_T [bs, C, H, W] (torch).  region_conds[r]:
    region r + 1's contexts (one per c_type); masks: latent masks fp64 [R, bs, H, W].  size: window side (None: one window, the
    canvas).  Bootstrapping at the first bootstrap_steps steps: pick_fn(i) -> int [R, bs] rows of backgrounds ([nb, C]),
    z_fn(i) -> z [bs, C, H, W].  With mask (latent, [bs or 1, 1, H, W]) and x0: the inpainting start and blend of inpaint_oracle,
    noise_fn(i) -> its z_i.  grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature).  The noise is the canvas's, added once per step: regions.py's step
    is the unchanged update on the mask-weighted eps average, so DDIM at eta > 0 takes that average and one canvas step."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    ts = sched["timesteps"]
    total = len(ts)
    H, W = x_T.shape[-2:]
    h, w, wins = P.windows(H, W, max(H, W) if size is None else size, max(H, W) if size is None else stride, circular)
    masks = np.asarray(masks, dtype=np.float64)
    acn = np.asarray(ac.numpy(), dtype=np.float64)
    x = I.start(x_T.float(), x0.float(), mask.float(), ac.numpy(), int(ts[-1])).float() if mask is not None else x_T.float()
    x = x.double().numpy()

    def boot_at(i):
        if i < total - bootstrap_steps:
            return None
        a = float(np.float32(np.sqrt(acn[ts[i]])))
        b = float(np.float32(np.sqrt(1.0 - acn[ts[i]])))
        bgs = np.asarray(backgrounds, dtype=np.float64)[np.asarray(pick_fn(i))]          # [R, bs, C]
        return bgs, np.asarray(z_fn(i), dtype=np.float64), a, b

    def views(xv, i, boot):
        xs = region_inputs(xv, masks, boot)
        return _views_eps(sd, xs, ts[i], conds, unconds, region_conds, wins, h, w, scale, c_types, ratios, kw)

    if sampler == "ddim":
        rows = I.blend_rows(ac.numpy(), ts).astype(np.float32)
        for i in range(total - 1, -1, -1):
            boot = boot_at(i)
            ev = views(x, i, boot)
            a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
            if eta == 0:
                x = paper_step(x, lambda xc, g, r: ev[g, r], masks, wins, h, w, a_t, a_prev, boot)
            else:
                e = eps_average(x, lambda xc, g, r: ev[g, r], masks, wins, h, w, boot)
                x = P.ddim_update(x, e, a_t, a_prev, float(sched["sigmas"][i]), np.asarray(noise(i), dtype=np.float64))
            if mask is not None:
                x = I.blend(torch.from_numpy(x).float(), x0.float(), mask.float(), noise_fn(i).float(), rows[i, 0],
                            rows[i, 1]).double().numpy()
        return torch.from_numpy(x).float()

    def eps_fn(xv, i):
        boot = boot_at(i)
        ev = views(np.asarray(xv, dtype=np.float64), i, boot)
        return eps_average(np.asarray(xv, dtype=np.float64), lambda xc, g, r: ev[g, r], masks, wins, h, w, boot)

    after = None if mask is None else I.blend_after(ac.numpy(), ts, x0, mask, noise_fn)
    out = G.dpm_walk(x, eps_fn, ac.numpy(), ts, order, eta, noise, after=after)
    return torch.from_numpy(out).float()
