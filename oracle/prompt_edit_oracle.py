"""Prompt-to-Prompt oracle — TEST INFRASTRUCTURE ONLY (never imported by the product path).

Restates lib/model_zoo/prompt_edit.py as P2P computes it: on materialised attention probabilities of vd_oracle.apply_model (the
fp32 UNet, with an attention hook on the text context's SpatialTransformers), with the mapper einsum, the equalizer
product, the alpha mix, the self-map replacement, and LocalBlend with max_pool2d / nearest interpolate.  It never forms the
factored A * ctx contexts, so comparing against it checks the factoring too.  The walk is DDIM or DPM-Solver++ (orders 1 to 3,
dpm_solver_oracle.walk with the local blend as its `after`) in fp64.
"""
import math

import torch
import torch.nn.functional as F

from . import dpm_sde_oracle as G
from . import panorama_oracle as P
from . import vd_oracle as O


class P2P(object):
    """The P2P controller over the CFG batch [uncond; cond] of n prompts.  kind 'replace' (M [n-1, L, L]), 'refine'
    (mp [n-1, L], alpha [n-1, L]) or 'reweight'; c [n-1, L] the equalizer; w [n, L] blend words or None."""

    def __init__(self, n, kind, T, cross_steps, self_steps, c, H, W, M=None, mp=None, alpha=None, w=None, threshold=0.3,
                 blend_start=0.0, cfg=True):
        self.n, self.kind, self.T, self.c, self.M, self.mp, self.alpha, self.w = n, kind, T, c, M, mp, alpha, w
        self.tc, self.ts = math.floor(cross_steps * T), math.floor(self_steps * T)
        self.tb, self.threshold, self.cfg = math.floor(blend_start * T), threshold, cfg
        self.h4, self.w4 = ((H + 1) // 2 + 1) // 2, ((W + 1) // 2 + 1) // 2
        self.i = 0
        self.maps = torch.zeros(n, self.h4 * self.w4, dtype=torch.float64)

    def hook(self, probs, cross):
        n = self.n
        c0 = n if self.cfg else 0
        N = probs.shape[2]
        cond = probs[c0:c0 + n]
        out = probs.clone()
        if cross:
            if self.w is not None and N == self.h4 * self.w4:      # the row's own probabilities, before the edit
                w = torch.as_tensor(self.w, dtype=torch.float64)
                self.maps += (cond.double() * w[:, None, None, :]).sum(dim=(1, 3))
            if self.i < self.tc:
                base = cond[0]
                for t in range(1, n):
                    c = torch.as_tensor(self.c[t - 1], dtype=probs.dtype)
                    if self.kind == "replace":
                        e = torch.einsum("hpw,wn->hpn", base, torch.as_tensor(self.M[t - 1], dtype=probs.dtype))
                    elif self.kind == "refine":
                        a = torch.as_tensor(self.alpha[t - 1], dtype=probs.dtype)
                        e = base[:, :, torch.as_tensor(self.mp[t - 1])] * a + cond[t] * (1 - a)
                    else:
                        e = base
                    out[c0 + t] = e * c
        elif N <= self.h4 * self.w4 and self.i < self.ts:
            for t in range(1, n):
                out[c0 + t] = cond[0]
        return out

    def blend(self, x):
        """LocalBlend after step i on x [n, C, H, W] (fp64)."""
        if self.w is None or self.i < self.tb:
            return x
        m = self.maps.view(self.n, 1, self.h4, self.w4)
        m = F.max_pool2d(m, (3, 3), (1, 1), padding=(1, 1))
        m = F.interpolate(m, size=x.shape[2:])
        mx = m.amax(dim=(2, 3), keepdim=True)
        m = torch.where(mx > 0, m / torch.where(mx > 0, mx, torch.ones_like(mx)), torch.zeros_like(m)).gt(self.threshold)
        m = m[:1] | m[1:]
        out = x.clone()
        out[1:] = torch.where(m, x[1:], x[:1])
        return out


def _eps_fn(sd, ctl, conds, unconds, scale, c_types, ratios, kw):
    def eps(x, t):
        tt = torch.full((x.shape[0],), int(t), dtype=torch.long)
        e_u, e_c = O.cfg_pass(O.apply_model, sd, x.float(), tt, conds, unconds, True, ratios, c_types,
                              hook_for=lambda j, idx: ctl.hook if c_types[j] == "text" else None, **kw)
        return e_u.double() + scale * (e_c.double() - e_u.double())
    return eps


def sample(sd, ctl, x_T, conds, unconds, steps, sampler="ddim", order=2, scale=7.5, c_types=("text",), ratios=None,
           num_ddpm=1000, grid_name="uniform", eta=0.0, noise=None, **kw):
    """The edited walk from x_T [n, C, H, W] (fp64 state, fp32 UNet) with the local blend after every step, over the first
    `steps` grid points (so over steps - 1 ... 0 also when a uniform grid has one more; a Karras grid can have fewer).  ctl.T
    is the walk's length.  grid_name: the sampler's time grid ('uniform', 'trailing' or 'karras'); eta: DDIM's eta, or the SDE walk's
    (dpm_sde_oracle.walk) for DPM-Solver++; noise(i) -> the step's standard normal z at grid index i, read where eta > 0 (for
    DDIM times the temperature)."""
    ac, sched = G.schedule(grid_name, steps, eta, num_ddpm)
    ts = sched["timesteps"][:steps]
    n = len(ts)
    eps = _eps_fn(sd, ctl, conds, unconds, scale, c_types, ratios, kw)
    x = x_T.double()
    if sampler == "ddim":
        for k, i in enumerate(range(n - 1, -1, -1)):
            ctl.i = k
            a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
            if eta == 0:
                x = P.ddim_update(x, eps(x, ts[i]), a_t, a_prev)
            else:
                x = P.ddim_update(x, eps(x, ts[i]), a_t, a_prev, float(sched["sigmas"][i]), torch.as_tensor(noise(i)).double())
            x = ctl.blend(x)
        return x

    def eps_fn(xv, i):
        ctl.i = n - 1 - i
        return eps(torch.from_numpy(xv), ts[i])

    out = G.dpm_walk(x.numpy(), eps_fn, ac.numpy(), ts, order, eta, noise,
                     after=lambda i, xn: ctl.blend(torch.from_numpy(xn)).numpy())
    return torch.from_numpy(out)
