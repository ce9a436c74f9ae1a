"""DPM-Solver++ multistep oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

An fp64 restatement of the deterministic multistep DPM-Solver++ (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling
of Diffusion Probabilistic Models", algorithm "dpmsolver++" of the paper's reference code, solver_type 'dpmsolver') on DDIM's
time grid.  Unlike lib/model_zoo/dpm_solver.py it never forms the folded per-step table: every step is taken directly from
lambda, expm1 and a list of earlier data predictions, so the tests can check the table against it.

Conventions shared with the product (see the module docstring of lib/model_zoo/dpm_solver.py):
  - alpha_i = sqrt(ac[t_i]), sigma_i = sqrt(1 - ac[t_i]), lambda_i = log alpha_i - log sigma_i, in fp64 from the fp32 buffer;
  - step i goes from t_i to t_{i-1}; step 0 goes to ac[0];
  - the walk visits i = len(timesteps) - 1, ..., 0; walk position k uses order min(order, k + 1), and when the walk has fewer
    than 15 steps also at most i + 1.
"""
import numpy as np
import torch

from . import vd_oracle as O


def coefficients(alphas_cumprod, timesteps):
    """fp64 (alpha, sigma, lambda) at every grid index, and (alpha', sigma') of each step's target."""
    ac = np.asarray(alphas_cumprod, dtype=np.float32).astype(np.float64)
    a = ac[np.asarray(timesteps)]
    alpha, sigma = np.sqrt(a), np.sqrt(1.0 - a)
    lam = np.log(alpha) - np.log(sigma)
    alpha_to = np.concatenate([[np.sqrt(ac[0])], alpha[:-1]])
    sigma_to = np.concatenate([[np.sqrt(1.0 - ac[0])], sigma[:-1]])
    return alpha, sigma, lam, alpha_to, sigma_to


def step_order(order, k, i, walk_len):
    o = min(order, k + 1)
    if walk_len < 15:
        o = min(o, i + 1)
    return o


def walk(x, eps_fn, alphas_cumprod, timesteps, order, trace=None):
    """fp64 multistep DPM-Solver++ from x (at t_{len-1}) down to ac[0].  eps_fn(x, i) -> the model's (CFG-mixed) eps at grid
    index i.  trace, when a list, receives (order, x0_i, x') per step."""
    alpha, sigma, lam, alpha_to, sigma_to = coefficients(alphas_cumprod, timesteps)
    n = len(timesteps)
    x = np.asarray(x, dtype=np.float64)
    x0s, lams = [], []
    for k, i in enumerate(range(n - 1, -1, -1)):
        x0 = (x - sigma[i] * np.asarray(eps_fn(x, i), dtype=np.float64)) / alpha[i]
        lam_to = np.log(alpha_to[i]) - np.log(sigma_to[i])
        h = lam_to - lam[i]
        phi1 = np.expm1(-h)
        o = step_order(order, k, i, n)
        xn = sigma_to[i] / sigma[i] * x - alpha_to[i] * phi1 * x0
        if o == 2:
            r0 = (lam[i] - lams[-1]) / h
            xn = xn - 0.5 * alpha_to[i] * phi1 * (x0 - x0s[-1]) / r0
        elif o == 3:
            r0, r1 = (lam[i] - lams[-1]) / h, (lams[-1] - lams[-2]) / h
            d1_0, d1_1 = (x0 - x0s[-1]) / r0, (x0s[-1] - x0s[-2]) / r1
            d1 = d1_0 + r0 / (r0 + r1) * (d1_0 - d1_1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            phi2 = phi1 / h + 1.0
            phi3 = phi2 / h - 0.5
            xn = xn + alpha_to[i] * phi2 * d1 - alpha_to[i] * phi3 * d2
        if trace is not None:
            trace.append((o, x0, xn))
        x0s.append(x0)
        lams.append(lam[i])
        x = xn
    return x


# ---- the analytic Gaussian model: data N(mu, s^2) per dimension --------------------------------------------------------------
def gaussian_eps(x, alpha, sigma, mu, s):
    """Exact eps of x_t = alpha x0 + sigma z with x0 ~ N(mu, s^2): E[z | x_t]."""
    return sigma * (x - alpha * mu) / (alpha * alpha * s * s + sigma * sigma)


def gaussian_exact(x_start, alpha_from, sigma_from, alpha_to, sigma_to, mu, s):
    """The probability-flow ODE solution: (x - alpha mu) / sqrt(alpha^2 s^2 + sigma^2) is constant along it."""
    m_from = np.sqrt(alpha_from ** 2 * s * s + sigma_from ** 2)
    m_to = np.sqrt(alpha_to ** 2 * s * s + sigma_to ** 2)
    return alpha_to * mu + (np.asarray(x_start, dtype=np.float64) - alpha_from * mu) * (m_to / m_from)


# ---- the mini-UNet walk: vd_oracle's fp32 UNet restatement + the fp64 solver --------------------------------------------------
def sample(sd, x_T, conds, unconds, steps, order, scale=7.5, c_types=("text",), ratios=None, text=False, num_ddpm=1000,
           x0=None, x0_forward_timesteps=None, x0_noise=None, **kw):
    """DPMSolverSampler.sample / sample_multicontext restated: DDIM's uniform grid and img2img start (vd_oracle.ddim_sample),
    the CFG mix e_u + scale (e_c - e_u) in fp32, the solver in fp64.  text: the [n, 768] latent through apply_model_text."""
    sch = O.ddpm_schedule(num_ddpm)
    ts = O.make_ddim_timesteps(steps, num_ddpm)
    x = x_T
    if x0 is not None:
        t0 = torch.full((x0.shape[0],), int(ts[x0_forward_timesteps]), dtype=torch.long)
        ts = ts[:x0_forward_timesteps]
        x = O.q_sample(x0, t0, x0_noise, num_ddpm)
    model = O.apply_model_text if text else O.apply_model

    def eps_fn(xv, i):
        xt = torch.from_numpy(np.asarray(xv)).float()
        t = torch.full((xt.shape[0],), int(ts[i]), dtype=torch.long)
        if scale == 1.0:
            return model(sd, xt, t, conds, ratios, c_types=c_types, **kw).double().numpy()
        c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
        e_u, e_c = model(sd, torch.cat([xt] * 2), torch.cat([t] * 2), c_in, ratios, c_types=c_types, **kw).chunk(2)
        return (e_u + scale * (e_c - e_u)).double().numpy()

    out = walk(x.double().numpy(), eps_fn, sch["alphas_cumprod"].numpy(), ts, order)
    return torch.from_numpy(out).float()
