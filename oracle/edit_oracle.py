"""Editing oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

An fp64 restatement of lib/model_zoo/edit.py: the inversion rows, the DDIM inversion walk (eps from vd_oracle.apply_model, the fp32
UNet restatement), the walk from an inversion with the trajectory blend after every step (DDIM, and DPM-Solver++ with the
steps of inpaint_oracle.dpm_walk and the trajectory in place of the re-noised x0), and DiffEdit's mask rule.
"""
import numpy as np
import torch

from . import dpm_solver_oracle as D
from . import vd_oracle as O


def inversion_rows(ddim_alphas, ddim_alphas_prev, k):
    """fp64 [k, 4] rows {a'_i, a_i, 0, sqrt(1 - a'_i)} of inversion steps 0 ... k-1."""
    a = np.asarray(ddim_alphas, dtype=np.float64)[:k]
    ap = np.asarray(ddim_alphas_prev, dtype=np.float64)[:k]
    return np.stack([ap, a, np.zeros_like(a), np.sqrt(1.0 - ap)], axis=1)


def _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw):
    def eps(x, t):
        tt = torch.full((x.shape[0],), int(t), dtype=torch.long)
        xf = x.float()
        if scale == 1.0:
            return O.apply_model(sd, xf, tt, conds, ratios, c_types=c_types, **kw).double()
        c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
        e_u, e_c = O.apply_model(sd, torch.cat([xf] * 2), torch.cat([tt] * 2), c_in, ratios, c_types=c_types, **kw).chunk(2)
        return (e_u.double() + scale * (e_c.double() - e_u.double()))
    return eps


def invert(sd, x0, conds, unconds, steps, k=None, scale=1.0, c_types=("text",), ratios=None, num_ddpm=1000, **kw):
    """The inversion walk in fp64 (eps from the fp32 UNet restatement) -> trajectory [k+1, bs, C, H, W] (slot 0 = x0)."""
    sched = O.ddim_schedule(O.ddpm_schedule(num_ddpm)["alphas_cumprod"], steps)
    ts = sched["timesteps"]
    k = len(ts) if k is None else k
    rows = inversion_rows(sched["alphas"], sched["alphas_prev"], k)
    eps = _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw)
    x = x0.double()
    traj = [x]
    for i in range(k):
        ap, a = rows[i, 0], rows[i, 1]
        e = eps(x, ts[i])
        x = np.sqrt(a) * (x - np.sqrt(1.0 - ap) * e) / np.sqrt(ap) + np.sqrt(1.0 - a) * e
        traj.append(x)
    return torch.stack(traj)


def sample(sd, traj, conds, unconds, steps, mask=None, sampler="ddim", order=2, scale=7.5, c_types=("text",), ratios=None,
           num_ddpm=1000, **kw):
    """The walk from slot k = len(traj) - 1 over grid points k-1 ... 0, with x <- m x + (1 - m) slot_i after step i when a
    latent mask [bs or 1, 1, H, W] is given (1 = regenerate)."""
    ac = O.ddpm_schedule(num_ddpm)["alphas_cumprod"]
    sched = O.ddim_schedule(ac, steps)
    k = traj.shape[0] - 1
    ts = sched["timesteps"][:k]
    m = None if mask is None else mask.double()
    eps = _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw)
    x = traj[k].double()
    if sampler == "ddim":
        for i in range(k - 1, -1, -1):
            a, ap = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
            e = eps(x, ts[i])
            x = np.sqrt(ap) * (x - np.sqrt(1.0 - a) * e) / np.sqrt(a) + np.sqrt(1.0 - ap) * e
            if m is not None:
                x = m * x + (1 - m) * traj[i].double()
        return x
    # DPM-Solver++: the steps of inpaint_oracle.dpm_walk, blended against slot i in place of x0 re-noised
    shape = x.shape
    mm = np.ones(shape) if m is None else m.expand(shape).numpy()
    slots = traj.double().numpy()
    alpha, sigma, lam, alpha_to, sigma_to = D.coefficients(ac.numpy(), ts)
    xv = x.numpy()
    x0s, lams = [], []
    for kk, i in enumerate(range(k - 1, -1, -1)):
        xp = (xv - sigma[i] * eps(torch.from_numpy(xv), ts[i]).numpy()) / alpha[i]
        h = np.log(alpha_to[i]) - np.log(sigma_to[i]) - lam[i]
        phi1 = np.expm1(-h)
        o = D.step_order(order, kk, i, k)
        xn = sigma_to[i] / sigma[i] * xv - alpha_to[i] * phi1 * xp
        if o == 2:
            r0 = (lam[i] - lams[-1]) / h
            xn = xn - 0.5 * alpha_to[i] * phi1 * (xp - x0s[-1]) / r0
        elif o == 3:
            r0, r1 = (lam[i] - lams[-1]) / h, (lams[-1] - lams[-2]) / h
            d1_0, d1_1 = (xp - x0s[-1]) / r0, (x0s[-1] - x0s[-2]) / r1
            d1 = d1_0 + r0 / (r0 + r1) * (d1_0 - d1_1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            phi2 = phi1 / h + 1.0
            phi3 = phi2 / h - 0.5
            xn = xn + alpha_to[i] * phi2 * d1 - alpha_to[i] * phi3 * d2
        xv = mm * xn + (1 - mm) * slots[i]
        x0s.append(xp)
        lams.append(lam[i])
    return torch.from_numpy(xv)


def diffedit_mask(e_src, e_tgt, ratio=3.0):
    """DiffEdit's rule in fp64.  e_src / e_tgt: the CFG-mixed eps [D, bs, C, H, W] -> {0, 1} [bs, 1, H, W] (and the distance)."""
    e_src, e_tgt = np.asarray(e_src, dtype=np.float64), np.asarray(e_tgt, dtype=np.float64)
    d = np.abs(e_tgt - e_src).mean(axis=(0, 2))                  # [bs, H, W]
    mu = d.reshape(d.shape[0], -1).mean(axis=1)[:, None, None]
    cap = ratio * mu
    with np.errstate(invalid="ignore", divide="ignore"):
        m = np.where(cap > 0, (np.minimum(d, cap) / cap >= 0.5), False).astype(np.float64)
    return m[:, None], d[:, None], cap[:, 0, 0]
