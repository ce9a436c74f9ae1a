"""Inpainting oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

A CPU restatement of the masked walk of lib/model_zoo/inpaint.py with the noises injected: DDIM through vd_oracle.p_sample_ddim
(the fp32 UNet restatement), DPM-Solver++ through the fp64 dpm_solver_oracle.walk (blend_after as its `after`), and after every
step the blend
    x' <- m x' + (1 - m) (sqrt(a') x0 + sqrt(1 - a') z_i)
with a' the cumulative alpha of the step's target (ac[t_{i-1}], ac[0] for i = 0) and the row {1, 0} at the last step.  The full
walk's start sets the kept region to sqrt(ac[t_top]) x0 + sqrt(1 - ac[t_top]) x_T.  Unlike the product it never builds the
device table: the rows come from the schedule here.
"""
import numpy as np
import torch

from . import dpm_sde_oracle as G
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


def blend_after(alphas_cumprod, timesteps, x0, mask, noise_fn):
    """The fp64 blend after step i as dpm_solver_oracle.walk's `after(i, x')`; noise_fn(i) -> z_i."""
    rows = blend_rows(alphas_cumprod, timesteps)
    x0, mask = np.asarray(x0, dtype=np.float64), np.asarray(mask, dtype=np.float64)
    return lambda i, x: blend(x, x0, mask, np.asarray(noise_fn(i), dtype=np.float64), rows[i, 0], rows[i, 1])


def sample(sd, x_T, conds, unconds, steps, x0, mask, noise_fn, sampler="ddim", order=2, scale=7.5, c_types=("text",),
           ratios=None, x0_forward_timesteps=None, x0_noise=None, num_ddpm=1000, grid_name="uniform", eta=0.0, noise=None, **kw):
    """The masked DDIMSampler / DPMSolverSampler walk on the UNet restatement.  x_T, x0 [bs or 1, C, H, W] and the latent mask
    [bs or 1, 1, H, W] as torch tensors; noise_fn(i) -> z_i, a [bs, C, H, W] tensor.  With x0_forward_timesteps the img2img start
    (x0 noised with x0_noise), else the full walk from x_T with the masked start.  grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature)."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    ts = sched["timesteps"]
    x0, mask = x0.float(), mask.float()
    if x0_forward_timesteps is not None:
        x, ts = O.img2img_start(x0, x0_noise, ts, x0_forward_timesteps, num_ddpm)
    else:
        x = start(x_T.float(), x0, mask, ac.numpy(), int(ts[-1])).float()
    if sampler == "ddim":
        rows = torch.from_numpy(blend_rows(ac.numpy(), ts).astype(np.float32))
        for i in range(len(ts) - 1, -1, -1):
            t = torch.full((x.shape[0],), int(ts[i]), dtype=torch.long)
            z = None if eta == 0 else torch.as_tensor(noise(i)).float()
            x, _, _ = O.p_sample_ddim(sd, x, conds, unconds, t, i, sched, scale, c_types, ratios, noise=z, **kw)
            x = blend(x, x0, mask, noise_fn(i).float(), rows[i, 0], rows[i, 1])
        return x

    def eps_fn(xv, i):
        t = torch.full((xv.shape[0],), int(ts[i]), dtype=torch.long)
        e_u, e_c = O.cfg_pass(O.apply_model, sd, torch.from_numpy(xv).float(), t, conds, unconds, scale != 1.0, ratios, c_types,
                              **kw)
        return (e_c if e_u is None else e_u + scale * (e_c - e_u)).double().numpy()

    out = G.dpm_walk(x.double().numpy(), eps_fn, ac.numpy(), ts, order, eta, noise,
                     after=blend_after(ac.numpy(), ts, x0, mask, noise_fn))
    return torch.from_numpy(out).float()
