"""Editing oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

An fp64 restatement of lib/model_zoo/edit.py: the inversion rows, the DDIM inversion walk (eps from vd_oracle.apply_model, the fp32
UNet restatement), the walk from an inversion with the trajectory blend after every step (DDIM, and dpm_solver_oracle.walk with
the blend against the trajectory as its `after`), and DiffEdit's mask rule.
"""
import numpy as np
import torch

from . import dpm_sde_oracle as G
from . import panorama_oracle as P
from . import vd_oracle as O


def inversion_rows(ddim_alphas, ddim_alphas_prev, k):
    """fp64 [k, 4] rows {a'_i, a_i, 0, sqrt(1 - a'_i)} of inversion steps 0 ... k-1."""
    a = np.asarray(ddim_alphas, dtype=np.float64)[:k]
    ap = np.asarray(ddim_alphas_prev, dtype=np.float64)[:k]
    return np.stack([ap, a, np.zeros_like(a), np.sqrt(1.0 - ap)], axis=1)


def _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw):
    def eps(x, t):
        tt = torch.full((x.shape[0],), int(t), dtype=torch.long)
        e_u, e_c = O.cfg_pass(O.apply_model, sd, x.float(), tt, conds, unconds, scale != 1.0, ratios, c_types, **kw)
        return e_c.double() if e_u is None else e_u.double() + scale * (e_c.double() - e_u.double())
    return eps


def invert(sd, x0, conds, unconds, steps, k=None, scale=1.0, c_types=("text",), ratios=None, num_ddpm=1000, grid_name="uniform",
           **kw):
    """The inversion walk in fp64 (eps from the fp32 UNet restatement) on grid grid_name -> trajectory [k+1, bs, C, H, W]
    (slot 0 = x0)."""
    sched = G.schedule(grid_name, steps, 0.0, num_ddpm)[1]
    ts = sched["timesteps"]
    k = len(ts) if k is None else k
    rows = inversion_rows(sched["alphas"], sched["alphas_prev"], k)
    eps = _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw)
    x = x0.double()
    traj = [x]
    for i in range(k):
        x = P.ddim_update(x, eps(x, ts[i]), rows[i, 0], rows[i, 1])
        traj.append(x)
    return torch.stack(traj)


def sample(sd, traj, conds, unconds, steps, mask=None, sampler="ddim", order=2, scale=7.5, c_types=("text",), ratios=None,
           num_ddpm=1000, grid_name="uniform", eta=0.0, noise=None, **kw):
    """The walk from slot k = len(traj) - 1 over grid points k-1 ... 0, with x <- m x + (1 - m) slot_i after step i when a
    latent mask [bs or 1, 1, H, W] is given (1 = regenerate).  grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature)."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    k = traj.shape[0] - 1
    ts = sched["timesteps"][:k]
    m = None if mask is None else mask.double()
    eps = _eps_fn(sd, conds, unconds, scale, c_types, ratios, kw)
    x = traj[k].double()
    if sampler == "ddim":
        for i in range(k - 1, -1, -1):
            a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
            if eta == 0:
                x = P.ddim_update(x, eps(x, ts[i]), a_t, a_prev)
            else:
                x = P.ddim_update(x, eps(x, ts[i]), a_t, a_prev, float(sched["sigmas"][i]), torch.as_tensor(noise(i)).double())
            if m is not None:
                x = m * x + (1 - m) * traj[i].double()
        return x
    mm, slots = None if m is None else m.numpy(), traj.double().numpy()
    after = None if mm is None else lambda i, xn: mm * xn + (1 - mm) * slots[i]
    out = G.dpm_walk(x.numpy(), lambda xv, i: eps(torch.from_numpy(xv), ts[i]), ac.numpy(), ts, order, eta, noise, after=after)
    return torch.from_numpy(out)


def diffedit_mask(e_src, e_tgt, ratio=3.0):
    """DiffEdit's rule in fp64.  e_src / e_tgt: the CFG-mixed eps [D, bs, C, H, W] -> {0, 1} [bs, 1, H, W] (and the distance)."""
    e_src, e_tgt = np.asarray(e_src, dtype=np.float64), np.asarray(e_tgt, dtype=np.float64)
    d = np.abs(e_tgt - e_src).mean(axis=(0, 2))                  # [bs, H, W]
    mu = d.reshape(d.shape[0], -1).mean(axis=1)[:, None, None]
    cap = ratio * mu
    with np.errstate(invalid="ignore", divide="ignore"):
        m = np.where(cap > 0, (np.minimum(d, cap) / cap >= 0.5), False).astype(np.float64)
    return m[:, None], d[:, None], cap[:, 0, 0]
