"""MultiDiffusion oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

A CPU restatement of the windowed walk of lib/model_zoo/panorama.py in the paper's form (Bar-Tal et al. 2023): every step crops
each window of the canvas, takes one step on the crop, and averages the windows' x_{t-1} per element.  DDIM runs through
vd_oracle.p_sample_ddim (the fp32 UNet restatement), with the windows' crops as one batch, and the average is taken in fp64.
DPM-Solver++ is a multistep method, so its paper form has no per-window state to average; it is the canvas walk of
dpm_solver_oracle.walk (with inpaint_oracle's blend as its `after` under a mask) with an eps function that averages the windows'
(CFG-mixed) eps.  The product averages eps in every case; the CPU test of the paper-form DDIM average against the eps average is
what checks that the two agree.

The layout is restated here independently of the product: sides min(size, L), origins 0, s, 2s, ... plus a final window flush
with the far edge (non-circular), or 0, s, ..., W - s with columns read mod W (circular, along W only).
"""
import numpy as np
import torch

from . import dpm_sde_oracle as G
from . import inpaint_oracle as I
from . import vd_oracle as O


def windows(H, W, size, stride, circular=False):
    """(h, w, [(oy, ox), ...] in window order: row-major over the origin grid)"""
    def axis(L, wrap):
        side = min(size, L)
        if wrap:
            return side, list(range(0, L, stride))
        o = list(range(0, L - side + 1, stride))
        return side, o if o[-1] == L - side else o + [L - side]
    h, oys = axis(H, False)
    w, oxs = axis(W, circular)
    return h, w, [(oy, ox) for oy in oys for ox in oxs]


def _cols(ox, w, W):
    return (ox + np.arange(w)) % W


def crop(x, oy, ox, h, w):
    """x[..., oy:oy+h, (ox + j) mod W]"""
    return x[..., oy:oy + h, :][..., _cols(ox, w, x.shape[-1])]


def average(parts, wins, h, w, shape):
    """fp64 per-element mean of the windows' arrays (each [..., h, w]) placed on a canvas of `shape`."""
    acc = np.zeros(shape, dtype=np.float64)
    cnt = np.zeros(shape[-2:], dtype=np.float64)
    W = shape[-1]
    for p, (oy, ox) in zip(parts, wins):
        cols = _cols(ox, w, W)
        acc[..., oy:oy + h, cols] += np.asarray(p, dtype=np.float64)
        cnt[oy:oy + h, cols] += 1
    return acc / cnt


def ddim_update(x, e, a_t, a_prev, sigma=0.0, z=None):
    """DDIM at eta 0: x' = sqrt(a') (x - sqrt(1 - a) e) / sqrt(a) + sqrt(1 - a') e.  With z (the step's standard normal times
    the temperature) the stochastic step of ddim.py:159-171: x' = sqrt(a') x0 + sqrt(1 - a' - sigma^2) e + sigma z."""
    if z is None:
        return np.sqrt(a_prev) * (x - np.sqrt(1.0 - a_t) * e) / np.sqrt(a_t) + np.sqrt(1.0 - a_prev) * e
    return np.sqrt(a_prev) * (x - np.sqrt(1.0 - a_t) * e) / np.sqrt(a_t) + np.sqrt(1.0 - a_prev - sigma ** 2) * e + sigma * z


def paper_step(x, eps_fn, wins, h, w, a_t, a_prev):
    """The paper's step: one DDIM step per window crop, then the per-element average of the windows' x_{t-1}.
    eps_fn(crop, window index) -> the crop's eps."""
    parts = []
    for g, (oy, ox) in enumerate(wins):
        xc = crop(x, oy, ox, h, w)
        parts.append(ddim_update(xc, eps_fn(xc, g), a_t, a_prev))
    return average(parts, wins, h, w, x.shape)


def eps_average(x, eps_fn, wins, h, w):
    """The product's form: the per-element average of the windows' eps."""
    return average([eps_fn(crop(x, oy, ox, h, w), g) for g, (oy, ox) in enumerate(wins)], wins, h, w, x.shape)


def _windowed_eps(sd, x, t, conds, unconds, wins, h, w, scale, c_types, ratios, kw):
    """the windows' CFG-mixed eps of x [bs, C, H, W] through the UNet restatement, averaged -> fp64 numpy canvas"""
    n, bs = len(wins), x.shape[0]
    xc = torch.cat([torch.from_numpy(crop(x.numpy(), oy, ox, h, w).copy()) for oy, ox in wins])      # row g*bs + b
    tt = torch.full((n * bs,), int(t), dtype=torch.long)
    rep = lambda cs: [c.repeat(n, 1, 1) for c in cs]
    e_u, e_c = O.cfg_pass(O.apply_model, sd, xc, tt, rep(conds), rep(unconds), scale != 1.0, ratios, c_types, **kw)
    e = e_c if e_u is None else e_u + scale * (e_c - e_u)
    e = e.double().numpy().reshape(n, bs, *e.shape[1:])
    return average(list(e), wins, h, w, x.shape)


def sample(sd, x_T, conds, unconds, steps, size, stride, circular=False, sampler="ddim", order=2, scale=7.5, c_types=("text",),
           ratios=None, x0=None, mask=None, noise_fn=None, x0_forward_timesteps=None, x0_noise=None, num_ddpm=1000,
           grid_name="uniform", eta=0.0, noise=None, **kw):
    """The windowed DDIMSampler / DPMSolverSampler walk on the UNet restatement.  x_T [bs, C, H, W] torch; with mask (latent,
    [bs or 1, 1, H, W]) the inpainting blend of inpaint_oracle after every step, noise_fn(i) -> z_i [bs, C, H, W]; with
    x0_forward_timesteps the img2img start (x0 noised with x0_noise), else the full walk from x_T (masked start with a mask).
    grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature).  The noise is the canvas's: DDIM at eta > 0 averages the windows' eps and takes one canvas step
    (lib/model_zoo/panorama.py and regions.py: the window walk is the region walk, whose step is the unchanged update on the
    averaged eps)."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    ts = sched["timesteps"]
    H, W = x_T.shape[-2:]
    h, w, wins = windows(H, W, size, stride, circular)
    if x0_forward_timesteps is not None:
        x, ts = O.img2img_start(x0.float(), x0_noise, ts, x0_forward_timesteps, num_ddpm)
    elif mask is not None:
        x = I.start(x_T.float(), x0.float(), mask.float(), ac.numpy(), int(ts[-1])).float()
    else:
        x = x_T.float()
    if sampler == "ddim":
        rows = torch.from_numpy(I.blend_rows(ac.numpy(), ts).astype(np.float32))
        for i in range(len(ts) - 1, -1, -1):
            if eta == 0:
                bs = x.shape[0]
                xc = torch.cat([torch.from_numpy(crop(x.numpy(), oy, ox, h, w).copy()) for oy, ox in wins])
                t = torch.full((xc.shape[0],), int(ts[i]), dtype=torch.long)
                rep = lambda cs: [c.repeat(len(wins), 1, 1) for c in cs]
                xp, _, _ = O.p_sample_ddim(sd, xc, rep(conds), rep(unconds), t, i, sched, scale, c_types, ratios, **kw)
                xp = xp.double().numpy().reshape(len(wins), bs, *xp.shape[1:])
                x = torch.from_numpy(average(list(xp), wins, h, w, x.shape)).float()
            else:
                e = _windowed_eps(sd, x, ts[i], conds, unconds, wins, h, w, scale, c_types, ratios, kw)
                x = torch.from_numpy(ddim_update(x.double().numpy(), e, float(sched["alphas"][i]), float(sched["alphas_prev"][i]),
                                                 float(sched["sigmas"][i]), np.asarray(noise(i), dtype=np.float64))).float()
            if mask is not None:
                x = I.blend(x, x0.float(), mask.float(), noise_fn(i).float(), rows[i, 0], rows[i, 1])
        return x

    def eps_fn(xv, i):
        return _windowed_eps(sd, torch.from_numpy(np.asarray(xv)).float(), ts[i], conds, unconds, wins, h, w, scale, c_types,
                             ratios, kw)

    after = None if mask is None else I.blend_after(ac.numpy(), ts, x0, mask, noise_fn)
    out = G.dpm_walk(x.double().numpy(), eps_fn, ac.numpy(), ts, order, eta, noise, after=after)
    return torch.from_numpy(out).float()
