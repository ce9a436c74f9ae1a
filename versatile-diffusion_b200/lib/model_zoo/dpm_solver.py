"""DPMSolverSampler — multistep DPM-Solver++ on the DDIM step graph, with the call surface of DDIMSampler.

The reference ships no such sampler; this is an addition.  Algorithm: Lu et al., "DPM-Solver++: Fast Solver for Guided Sampling
of Diffusion Probabilistic Models" (2022), the deterministic multistep "dpmsolver++" update of the paper's reference code
(solver_type 'dpmsolver').  One UNet evaluation per step, as DDIM, with an error that falls as h^order instead of h.

Schedule.  DDIM's 'uniform' grid t_i (make_ddim_timesteps) and the model's fp32 alphas_cumprod buffer `ac`, evaluated in fp64:
    alpha_i = sqrt(ac[t_i]),  sigma_i = sqrt(1 - ac[t_i]),  lambda_i = log alpha_i - log sigma_i.
Step i goes from t_i to t_{i-1}; step 0 goes to ac[0] (DDIM's alphas_prev).  The walk visits the same indices as DDIM,
total-1, ..., 0, with DDIMSampler._initial_latent's img2img start (x0 noised to t_k, then the first k grid points).

Model output.  e = e_u + s (e_c - e_u) (the CFG mix of vdb_ddim_cfg_step), data prediction x0_i = (x - sigma_i e) / alpha_i.

Update, with primes for the target point:  h = lambda' - lambda_i,  phi1 = expm1(-h).
    order 1:  x' = (sigma'/sigma_i) x - alpha' phi1 x0_i                                  (equal to DDIM at eta 0)
    order 2:  r0 = (lambda_i - lambda_{i+1}) / h,  D = (1 + 1/(2 r0)) x0_i - x0_{i+1} / (2 r0),
              x' = (sigma'/sigma_i) x - alpha' phi1 D
    order 3:  r1 = (lambda_{i+1} - lambda_{i+2}) / h,  D1_0 = (x0_i - x0_{i+1}) / r0,  D1_1 = (x0_{i+1} - x0_{i+2}) / r1,
              D1 = D1_0 + r0/(r0 + r1) (D1_0 - D1_1),  D2 = (D1_0 - D1_1) / (r0 + r1),
              phi2 = phi1/h + 1,  phi3 = phi2/h - 0.5,
              x' = (sigma'/sigma_i) x - alpha' phi1 x0_i + alpha' phi2 D1 - alpha' phi3 D2
Order per step.  Walk position k (0-based) at index i uses order min(order, k + 1): the first steps warm up on the history they
have.  When the walk has fewer than 15 steps the order is also at most i + 1, so the last steps drop to lower order.  The walk
is DDIM's: range(0, 1000, 1000 // steps) + 1, so a step count that does not divide 1000 walks more points (14 steps walk 15).

Folding.  All of it is linear in (x, e, x0_i, x0_{i+1}, x0_{i+2}), so each step is one table row {P, Q, A, B, C, D, 0, 0}
built on the host in fp64 and stored as fp32 (dpmpp_table):
    x0 = P x + Q e,   x' = A x + B x0_i + C x0_{i+1} + D x0_{i+2}.
The device keeps x0 of the last three steps in a ring (slot idx % 3), so vdb_dpmpp_cfg_step replaces vdb_ddim_cfg_step in
DDIMSampler's captured step graph and every step, warm-up and final steps included, is one replay of it.

Differences from DDIMSampler: eta != 0 raises ValueError (no stochastic variant); temperature and noise_dropout have no effect
(as in DDIM at eta 0); p_sample_ddim / p_sample_ddim_multicontext raise NotImplementedError (a multistep solver has no
single-step form).  order in {1, 2, 3}; the default 2 is the paper's recommendation for guided sampling.
"""
import numpy as np
import torch

from .ddim import DDIMSampler


def _ops():
    from vdb200 import ops
    return ops


def step_order(order, k, i, walk_len):
    """Solver order at walk position k (0-based) with grid index i, for a walk of walk_len steps."""
    o = min(order, k + 1)
    if walk_len < 15:
        o = min(o, i + 1)
    return o


def dpmpp_table(alphas_cumprod, timesteps, order):
    """fp64 [len(timesteps), 8] rows {P, Q, A, B, C, D, 0, 0}, indexed by the grid index i, for the walk over `timesteps`
    (the grid points actually visited: DDIM's ddim_timesteps, shortened by an img2img start)."""
    if order not in (1, 2, 3):
        raise ValueError(f"order must be 1, 2 or 3, got {order!r}")
    ac = np.asarray(alphas_cumprod.cpu() if isinstance(alphas_cumprod, torch.Tensor) else alphas_cumprod,
                    dtype=np.float32).astype(np.float64)
    ts = np.asarray(timesteps)
    n = ts.shape[0]
    alpha, sigma = np.sqrt(ac[ts]), np.sqrt(1.0 - ac[ts])
    lam = np.log(alpha) - np.log(sigma)
    alpha_to = np.concatenate([[np.sqrt(ac[0])], alpha[:-1]])
    sigma_to = np.concatenate([[np.sqrt(1.0 - ac[0])], sigma[:-1]])
    lam_to = np.log(alpha_to) - np.log(sigma_to)
    table = np.zeros((n, 8), dtype=np.float64)
    for i in range(n):
        k = n - 1 - i
        h = lam_to[i] - lam[i]
        phi1 = np.expm1(-h)
        a_ = alpha_to[i]
        # coefficients of x0_i, x0_{i+1}, x0_{i+2} in x'
        m = np.array([-a_ * phi1, 0.0, 0.0])
        o = step_order(order, k, i, n)
        if o == 2:
            r0 = (lam[i] - lam[i + 1]) / h
            m += -a_ * phi1 * np.array([1.0, -1.0, 0.0]) / (2.0 * r0)
        elif o == 3:
            r0, r1 = (lam[i] - lam[i + 1]) / h, (lam[i + 1] - lam[i + 2]) / h
            d1_0 = np.array([1.0, -1.0, 0.0]) / r0
            d1_1 = np.array([0.0, 1.0, -1.0]) / r1
            d1 = d1_0 + r0 / (r0 + r1) * (d1_0 - d1_1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            phi2 = phi1 / h + 1.0
            phi3 = phi2 / h - 0.5
            m += a_ * phi2 * d1 - a_ * phi3 * d2
        table[i, :6] = [1.0 / alpha[i], -sigma[i] / alpha[i], sigma_to[i] / sigma[i], m[0], m[1], m[2]]
    return table


class DPMSolverSampler(DDIMSampler):
    _coef_cols = 8

    def __init__(self, model, schedule="linear", order=2, **kwargs):
        if order not in (1, 2, 3):
            raise ValueError(f"DPMSolverSampler: order must be 1, 2 or 3, got {order!r}")
        super().__init__(model, schedule=schedule, **kwargs)
        self.order = order

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        if ddim_eta != 0:
            raise ValueError('ddim_eta must be 0 for DPM-Solver++')
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)

    def _coef_table(self, timesteps, sigmas):
        return dpmpp_table(self.model.alphas_cumprod, timesteps, self.order)

    def _state(self, bs, B, H, W, C, device):
        st = super()._state(bs, B, H, W, C, device)
        if 'hist' not in st:
            st['hist'] = torch.zeros(3 * bs * H * W * C, dtype=torch.float32, device=device)
        return st

    def _update(self, st, e_u, e_c, scale, bs, cfg, noise, temperature):
        _ops().dpmpp_cfg_step(e_u, e_c, st['x_in'][:bs], st['coef'], st['idx'], scale, st['hist'], x_next=st['x_in'][:bs],
                              x_next_dup=st['x_in'][bs:] if cfg else None, pred_x0=st['pred_x0'])

    def _graph_tag(self):
        return ('dpmpp', self.order)

    def p_sample_ddim(self, *args, **kwargs):
        raise NotImplementedError("DPMSolverSampler is a multistep solver: it has no single-step form (use sample)")

    def p_sample_ddim_multicontext(self, *args, **kwargs):
        raise NotImplementedError("DPMSolverSampler is a multistep solver: it has no single-step form (use sample_multicontext)")
