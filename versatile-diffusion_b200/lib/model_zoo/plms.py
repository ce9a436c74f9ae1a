"""PLMSSampler — pseudo linear multi-step sampling on the same VD_v2_0.apply_model hot path.

The reference ships NO PLMS sampler; BASELINE.json's north star names one, so this is an
ADDITION with the call surface of DDIMSampler (`sample`, `sample_multicontext`).  Algorithm: Liu et al., "Pseudo
Numerical Methods for Diffusion Models on Manifolds" (ICLR 2022) as used by CompVis latent-diffusion's plms.py —
eps history combined with Adams-Bashforth weights, first step by a pseudo improved-Euler (two model calls):
    e' = e_t                                   (+ e(x_prev, t_next))/2      first step
    e' = (3 e_t - e_{t-1}) / 2                                               second
    e' = (23 e_t - 16 e_{t-1} + 5 e_{t-2}) / 12                              third
    e' = (55 e_t - 59 e_{t-1} + 37 e_{t-2} - 9 e_{t-3}) / 24                 afterwards
followed by the eta = 0 DDIM update with e'.  Parity is pinned to the oracle restatement
(oracle/vd_oracle.py:plms_sample) only — there is no reference implementation to compare with.
Kernels: the UNet walk, `vdb_ddim_cfg_step` (CFG mix -> fp32 eps, and the x_{t-1} update) and `vdb_lincomb4_f32`.
"""
import numpy as np
import torch

from .ddim import DDIMSampler
from .diffusion_utils import to_numpy


def _ops():
    from vdb200 import ops
    return ops


class PLMSSampler(DDIMSampler):
    def __init__(self, model, schedule="linear", **kwargs):
        kwargs.setdefault("use_cuda_graph", False)
        super().__init__(model, schedule=schedule, **kwargs)

    def make_schedule(self, ddim_num_steps, ddim_discretize=None, ddim_eta=0., verbose=True):
        if ddim_eta != 0:
            raise ValueError('ddim_eta must be 0 for PLMS')
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)

    def invert(self, *args, **kwargs):
        raise NotImplementedError("PLMSSampler has no inversion: invert with DDIMSampler (lib/model_zoo/edit.py)")

    def invert_multicontext(self, *args, **kwargs):
        self.invert()

    def _run(self, shape, x_info, c_infos, multi, noise_dropout, temperature, log_every_t):
        self._modes('plms', x_info, shape, c_infos)
        ops = _ops()
        model = self.model
        device = torch.device(model.device)
        if device.type != 'cuda':
            raise RuntimeError("PLMSSampler: the H100 build has no CPU path (model.to('cuda') first)")
        dtype = c_infos[0]['conditioning'].dtype
        bs = shape[0]
        x, timesteps = self._initial_latent(shape, x_info, dtype, device)
        scale = float(c_infos[0]['unconditional_guidance_scale'])
        cfg = scale != 1.
        total = timesteps.shape[0]
        x_type = x_info['type']
        ctxs, c_types, ratios, time_from, mch = self._contexts(c_infos, cfg, x_type, multi)
        B = 2 * bs if cfg else bs
        coef = torch.tensor(self._coef_table(timesteps, to_numpy(self.ddim_sigmas)), dtype=torch.float32, device=device)
        # identity coefficients turn vdb_ddim_cfg_step into a pure CFG mix: a_t = 1, a_prev = 1, sigma = 0,
        # sqrt(1-a_t) = -1  =>  pred_x0 = x + e  with x = 0, i.e. pred_x0 = e_u + s (e_c - e_u)
        ident = torch.tensor([[1.0, 1.0, 0.0, -1.0]], dtype=torch.float32, device=device)

        xh = ops.nchw_to_nhwc(x.float().contiguous())
        x_in = torch.empty((B,) + tuple(xh.shape[1:]), dtype=torch.float32, device=device)
        zeros = torch.zeros_like(xh)

        def model_eps(x_nhwc, step_value):
            """CFG-mixed fp32 eps (NHWC) of the model at one timestep."""
            x_in[:bs].copy_(x_nhwc)
            if cfg:
                x_in[bs:].copy_(x_nhwc)
            ts = torch.full((B,), int(step_value), dtype=torch.int64, device=device)
            t_emb = ops.timestep_embedding(ts, mch)
            eps = model.eps_nhwc(x_in, x_type, t_emb, c_types, ctxs, ratios, time_from)
            if not cfg:
                return eps
            e = torch.empty_like(x_nhwc)
            ops.ddim_cfg_step(eps[:bs], eps[bs:], zeros, ident, scale, x_prev=torch.empty_like(x_nhwc), pred_x0=e)
            return e

        def update(x_nhwc, e, index):
            x_prev, pred_x0 = torch.empty_like(x_nhwc), torch.empty_like(x_nhwc)
            ops.ddim_cfg_step(None, e, x_nhwc, coef[index:index + 1].contiguous(), 1.0, x_prev=x_prev, pred_x0=pred_x0)
            return x_prev, pred_x0

        intermediates = {'pred_xt': [], 'pred_x0': []}
        old_eps = []
        time_range = np.flip(timesteps)
        for i, step in enumerate(time_range):
            index = total - i - 1
            step_next = time_range[min(i + 1, total - 1)]
            e_t = model_eps(xh, step)
            if len(old_eps) == 0:
                x_prev, _ = update(xh, e_t, index)
                e_next = model_eps(x_prev, step_next)
                e_prime = ops.lincomb4([e_t, e_next], [0.5, 0.5])
            elif len(old_eps) == 1:
                e_prime = ops.lincomb4([e_t, old_eps[-1]], [1.5, -0.5])
            elif len(old_eps) == 2:
                e_prime = ops.lincomb4([e_t, old_eps[-1], old_eps[-2]], [23. / 12, -16. / 12, 5. / 12])
            else:
                e_prime = ops.lincomb4([e_t, old_eps[-1], old_eps[-2], old_eps[-3]], [55. / 24, -59. / 24, 37. / 24, -9. / 24])
            xh, pred_x0 = update(xh, e_prime, index)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
            if index % log_every_t == 0 or index == total - 1:
                intermediates['pred_xt'].append(ops.nhwc_to_nchw(xh).to(dtype))
                intermediates['pred_x0'].append(ops.nhwc_to_nchw(pred_x0).to(dtype))
        out = ops.nhwc_to_nchw(xh).to(dtype)
        x_info['x'] = out
        return out, intermediates
