"""Inpainting oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

A CPU restatement of the masked walk of lib/model_zoo/inpaint.py with the noises injected: DDIM through vd_oracle.p_sample_ddim
(the fp32 UNet restatement), DPM-Solver++ through the fp64 steps of oracle/dpm_solver_oracle.py, and after every step the blend
    x' <- m x' + (1 - m) (sqrt(a') x0 + sqrt(1 - a') z_i)
with a' the cumulative alpha of the step's target (ac[t_{i-1}], ac[0] for i = 0) and the row {1, 0} at the last step.  The full
walk's start sets the kept region to sqrt(ac[t_top]) x0 + sqrt(1 - ac[t_top]) x_T.  Unlike the product it never builds the
device table: the rows come from the schedule here.
"""
import numpy as np
import torch

from . import dpm_solver_oracle as D
from . import vd_oracle as O


def blend_rows(alphas_cumprod, timesteps):
    """fp64 [len(timesteps), 2]: {sqrt(a'), sqrt(1 - a')} of each step's target; row 0 is {1, 0}."""
    ac = np.asarray(alphas_cumprod, dtype=np.float32).astype(np.float64)
    ts = np.asarray(timesteps)
    a_to = np.concatenate([[ac[0]], ac[ts[:-1]]])
    rows = np.stack([np.sqrt(a_to), np.sqrt(1.0 - a_to)], axis=1)
    rows[0] = (1.0, 0.0)
    return rows


def blend(x, x0, mask, z, a, b):
    return mask * x + (1 - mask) * (a * x0 + b * z)


def start(x_T, x0, mask, alphas_cumprod, t_top):
    """the full walk's start: the kept region of x_T becomes x0 noised to t_top with x_T's own draw"""
    a = float(np.float32(np.asarray(alphas_cumprod, dtype=np.float32)[t_top]))
    return blend(x_T, x0, mask, x_T, np.sqrt(a), np.sqrt(1.0 - a))


def dpm_walk(x, eps_fn, alphas_cumprod, timesteps, order, x0, mask, noise_fn, trace=None):
    """fp64 multistep DPM-Solver++ (dpm_solver_oracle.walk's steps; order 1 is DDIM at eta 0) from x at t_{len-1}, with the blend
    after every step.  noise_fn(i) -> z_i.  trace, when a list, receives x' after each blend."""
    alpha, sigma, lam, alpha_to, sigma_to = D.coefficients(alphas_cumprod, timesteps)
    rows = blend_rows(alphas_cumprod, timesteps)
    n = len(timesteps)
    x = np.asarray(x, dtype=np.float64)
    x0s, lams = [], []
    for k, i in enumerate(range(n - 1, -1, -1)):
        xp = (x - sigma[i] * np.asarray(eps_fn(x, i), dtype=np.float64)) / alpha[i]
        h = np.log(alpha_to[i]) - np.log(sigma_to[i]) - lam[i]
        phi1 = np.expm1(-h)
        o = D.step_order(order, k, i, n)
        xn = sigma_to[i] / sigma[i] * x - alpha_to[i] * phi1 * xp
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
        x = blend(xn, x0, mask, np.asarray(noise_fn(i), dtype=np.float64), rows[i, 0], rows[i, 1])
        if trace is not None:
            trace.append(x)
        x0s.append(xp)
        lams.append(lam[i])
    return x


def sample(sd, x_T, conds, unconds, steps, x0, mask, noise_fn, sampler="ddim", order=2, scale=7.5, c_types=("text",),
           ratios=None, x0_forward_timesteps=None, x0_noise=None, num_ddpm=1000, **kw):
    """The masked DDIMSampler / DPMSolverSampler walk on the UNet restatement.  x_T, x0 [bs or 1, C, H, W] and the latent mask
    [bs or 1, 1, H, W] as torch tensors; noise_fn(i) -> z_i, a [bs, C, H, W] tensor.  With x0_forward_timesteps the img2img start
    (x0 noised with x0_noise), else the full walk from x_T with the masked start."""
    ac = O.ddpm_schedule(num_ddpm)["alphas_cumprod"]
    sched = O.ddim_schedule(ac, steps)
    ts = sched["timesteps"]
    x0, mask = x0.float(), mask.float()
    if x0_forward_timesteps is not None:
        t0 = torch.full((x0.shape[0],), int(ts[x0_forward_timesteps]), dtype=torch.long)
        ts = ts[:x0_forward_timesteps]
        x = O.q_sample(x0, t0, x0_noise, num_ddpm)
    else:
        x = start(x_T.float(), x0, mask, ac.numpy(), int(ts[-1])).float()
    if sampler == "ddim":
        rows = torch.from_numpy(blend_rows(ac.numpy(), ts).astype(np.float32))
        for i in range(len(ts) - 1, -1, -1):
            t = torch.full((x.shape[0],), int(ts[i]), dtype=torch.long)
            x, _, _ = O.p_sample_ddim(sd, x, conds, unconds, t, i, sched, scale, c_types, ratios, **kw)
            x = blend(x, x0, mask, noise_fn(i).float(), rows[i, 0], rows[i, 1])
        return x

    def eps_fn(xv, i):
        xt = torch.from_numpy(np.asarray(xv)).float()
        t = torch.full((xt.shape[0],), int(ts[i]), dtype=torch.long)
        if scale == 1.0:
            return O.apply_model(sd, xt, t, conds, ratios, c_types=c_types, **kw).double().numpy()
        c_in = [torch.cat([u, c]) for u, c in zip(unconds, conds)]
        e_u, e_c = O.apply_model(sd, torch.cat([xt] * 2), torch.cat([t] * 2), c_in, ratios, c_types=c_types, **kw).chunk(2)
        return (e_u + scale * (e_c - e_u)).double().numpy()

    out = dpm_walk(x.double().numpy(), eps_fn, ac.numpy(), ts, order, x0.double().numpy(), mask.double().numpy(),
                   lambda i: noise_fn(i).double().numpy())
    return torch.from_numpy(out).float()
