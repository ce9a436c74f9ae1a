"""Stochastic DPM-Solver++ and the trailing / Karras time grids, restated for the tests in fp64 — never imported by the product.

Like dpm_solver_oracle.py, whose conventions and helpers it reuses, the SDE step here is taken directly from lambda, expm1
and the list of earlier data predictions, never from the folded table of lib/model_zoo/dpm_solver.py.  At eta = 0 the step is
dpm_solver_oracle.walk's.  The grids are restated from their sources, not from make_ddim_timesteps:
  - trailing: diffusers' DDIMScheduler / DPMSolverMultistepScheduler, timestep_spacing="trailing":
        np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
    np.arange's length is computed in floating point and comes out as n + 1 for some n (61, 103, ...): the extra point lies at
    about 0 and rounds to t = -1.  The grid is the first n points.
  - karras: k-diffusion's get_sigmas_karras (rho = 7, torch.linspace ramp) between sigma(T - 1) and sigma(1), mapped to t by
    diffusers' _sigma_to_t over log sigma(t), sigma(t) = ((1 - ac) / ac) ** 0.5 from the fp32 buffer; np.rint, repeats dropped.
"""
import numpy as np
import torch

from . import dpm_solver_oracle as D
from . import vd_oracle as O


def trailing_grid(n, T=1000):
    return np.sort((np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1)[:n])


def _sigma_to_t(sigma, log_sigmas):
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    return (1 - w) * low_idx + w * high_idx


def karras_grid(alphas_cumprod, n, rho=7.0):
    ac = np.asarray(alphas_cumprod, dtype=np.float32).astype(np.float64)
    sigmas_t = ((1 - ac) / ac) ** 0.5
    ramp = torch.linspace(0, 1, n, dtype=torch.float64).numpy()
    min_inv_rho, max_inv_rho = sigmas_t[1] ** (1 / rho), sigmas_t[-1] ** (1 / rho)
    sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
    return np.unique(np.rint(_sigma_to_t(sigmas, np.log(sigmas_t))).astype(np.int64))


def grid(name, n, alphas_cumprod, T=1000):
    if name == "uniform":
        return O.make_ddim_timesteps(n, T)
    return trailing_grid(n, T) if name == "trailing" else karras_grid(alphas_cumprod, n)


def walk(x, eps_fn, alphas_cumprod, timesteps, order, eta=0.0, noise=None, trace=None, after=None):
    """fp64 multistep DPM-Solver++ (SDE form for eta > 0) from x at t_{len-1} down to ac[0].  noise(i) -> z of step i (standard
    normals shaped like x), read only where eta_i > 0; eta_i = eta except at i = 0, where the step is deterministic.  eps_fn,
    after and trace as dpm_solver_oracle.walk; trace also receives z (or None)."""
    alpha, sigma, lam, alpha_to, sigma_to = D.coefficients(alphas_cumprod, timesteps)
    n = len(timesteps)
    x = np.asarray(x, dtype=np.float64)
    x0s, lams = [], []
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = (x - sigma[i] * np.asarray(eps_fn(x, i), dtype=np.float64)) / alpha[i]
        lam_to = np.log(alpha_to[i]) - np.log(sigma_to[i])
        h = lam_to - lam[i]
        e = eta if i > 0 else 0.0
        he = (1.0 + e) * h
        xn = sigma_to[i] / sigma[i] * np.exp(-e * h) * x + alpha_to[i] * -np.expm1(-he) * x0
        o = D.step_order(order, k, i, n)
        if o == 2:
            r0 = (lam[i] - lams[-1]) / h
            xn = xn + 0.5 * alpha_to[i] * -np.expm1(-he) / r0 * (x0 - x0s[-1])
        elif o == 3:
            r0, r1 = (lam[i] - lams[-1]) / h, (lams[-1] - lams[-2]) / h
            d1_0, d1_1 = (x0 - x0s[-1]) / r0, (x0s[-1] - x0s[-2]) / r1
            d1 = d1_0 + (d1_0 - d1_1) * r0 / (r0 + r1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            phi2 = np.expm1(-he) / he + 1.0
            phi3 = phi2 / he - 0.5
            xn = xn + alpha_to[i] * (phi2 * d1 - phi3 * d2)
        z = None
        if e > 0:
            z = np.asarray(noise(i), dtype=np.float64)
            xn = xn + sigma_to[i] * np.sqrt(-np.expm1(-2.0 * e * h)) * z
        if trace is not None:
            trace.append((o, x0, xn, z))
        x0s.append(x0)
        lams.append(lam[i])
        x = xn if after is None else after(i, xn)
    return x


def dpm_walk(x, eps_fn, alphas_cumprod, timesteps, order, eta=0.0, noise=None, after=None):
    """The feature oracles' DPM-Solver++ walk: dpm_solver_oracle.walk at eta = 0 (so their default outputs keep its op grouping
    bit for bit), else the SDE walk above."""
    if eta == 0:
        return D.walk(x, eps_fn, alphas_cumprod, timesteps, order, after=after)
    return walk(x, eps_fn, alphas_cumprod, timesteps, order, eta=eta, noise=noise, after=after)


def schedule(name, steps, eta=0.0, num_ddpm=1000):
    """vd_oracle.ddim_schedule with DDIM's sigmas at eta on grid `name` -> (the fp32 alphas_cumprod tensor, the schedule)."""
    ac = O.ddpm_schedule(num_ddpm)["alphas_cumprod"]
    return ac, O.ddim_schedule(ac, steps, eta, timesteps=None if name == "uniform" else grid(name, steps, ac.numpy(), num_ddpm))


def sample(sd, x_T, conds, unconds, steps, order, scale=7.5, c_types=("text",), ratios=None, text=False, num_ddpm=1000,
           x0=None, x0_forward_timesteps=None, x0_noise=None, grid_name="uniform", eta=0.0, noise=None, **kw):
    """DPMSolverSDESampler.sample / sample_multicontext (DPMSolverSampler's at eta = 0) restated on the mini UNet: the grid, the
    img2img start, vd_oracle's fp32 UNet and CFG pass, the solver in fp64.  noise(i) -> the step's z (NCHW, or [n, 768])."""
    sch = O.ddpm_schedule(num_ddpm)
    ac = sch["alphas_cumprod"].numpy()
    ts = grid(grid_name, steps, ac, num_ddpm)
    x = x_T
    if x0 is not None:
        x, ts = O.img2img_start(x0, x0_noise, ts, x0_forward_timesteps, num_ddpm)
    model = O.apply_model_text if text else O.apply_model

    def eps_fn(xv, i):
        t = torch.full((xv.shape[0],), int(ts[i]), dtype=torch.long)
        e_u, e_c = O.cfg_pass(model, sd, torch.from_numpy(xv).float(), t, conds, unconds, scale != 1.0, ratios, c_types, **kw)
        return (e_c if e_u is None else e_u + scale * (e_c - e_u)).double().numpy()

    out = walk(x.double().numpy(), eps_fn, ac, ts, order, eta=eta, noise=noise)
    return torch.from_numpy(out).float()
