"""Semantic/style disentanglement of the image context — `decompose` and `adjust_rank` of the reference app.py:48-127, the
"focus" slider (fcs_lvl) of the i2i, dcg, mcg and tcg flows.

`adjust_rank(max_drop_rank, q)(x, lvl)` takes the [n, m, 768] local CLIP image tokens and returns them with the leading singular
values of each item scaled down (lvl < 0.5: semantics) or the trailing ones (lvl > 0.5: style), rescaled to the item's standard
deviation.  The randomized PCA, the rescaling and the reconstruction run as one kernel launch (`vdb_rank_adjust_f32`); only the
factor schedule is computed here, on the host.  Differences from the reference:
  - every item of the batch gets its own standard deviation (the reference broadcasts the [n] std vector against the feature
    axis, so it only runs for n = 1, where both agree);
  - the QRs are CholeskyQR2 rather than Householder, so U and V may differ from torch.pca_lowrank's by the signs of their
    columns; S and every output of adjust_rank are sign-free.
The Gaussian start is drawn as torch.pca_lowrank draws it (`torch.randn(m, q)` on x's device from its default generator), so a
seeded call uses the reference's start and leaves the generator where the reference leaves it; `R=` passes it explicitly (tests,
CUDA-graph capture).
"""
import numpy as np
import torch

from vdb200 import ops

from .diffusion_utils import require_cuda


def _start(x, q, R):
    if R is None:
        return torch.randn(x.shape[-2], q, dtype=torch.float32, device=x.device)
    return R.to(device=x.device, dtype=torch.float32).contiguous()


def decompose(x, q=20, niter=100, R=None):
    """app.py's decompose: (u [n,m,q], s [n,q], v [n,768,q], x_mean [n,m,1], x_remain [n,m,768]) of fp32 x [n, m, 768]."""
    require_cuda(x, "decompose")
    x = x.float().contiguous()
    n, m, d = x.shape
    s = torch.empty(n, q, dtype=torch.float32, device=x.device)
    u = torch.empty(n, m, q, dtype=torch.float32, device=x.device)
    v = torch.empty(n, d, q, dtype=torch.float32, device=x.device)
    ops.rank_adjust(x, torch.ones(q, dtype=torch.float32, device=x.device), True, _start(x, q, R), niter=niter, s_out=s,
                    u_out=u, v_out=v)
    x_mean = x.mean(-1, keepdim=True)
    x_remain = (x - x_mean) - torch.bmm(u * s[:, None, :], v.transpose(1, 2))
    return u, s, v, x_mean, x_remain


class adjust_rank(object):
    def __init__(self, max_drop_rank=[1, 5], q=20):
        self.max_semantic_drop_rank = max_drop_rank[0]
        self.max_style_drop_rank = max_drop_rank[1]
        self.q = q
        self.niter = 100

    def factors(self, lvl):
        """The factor applied to each of the q singular values at focus level lvl (app.py:63-114), as float64."""
        f = np.ones(self.q)
        centre = np.exp((0.5 - 0.5) * 2)
        if lvl < 0.5:
            assert lvl >= 0
            t0, y00, x1 = np.exp((0 - 0.5) * 2), -self.max_semantic_drop_rank, self.max_semantic_drop_rank + 1
            y0 = (np.exp((lvl - 0.5) * 2) - t0) / (centre - t0) * (1 - y00) + y00
            for xi in range(0, self.max_semantic_drop_rank + 1):
                f[xi] = max((xi - 0) / (x1 - 0) * (1 - y0) + y0, 0)
        elif lvl > 0.5:
            assert lvl <= 1
            t0, y00 = np.exp((1 - 0.5) * 2), -(self.q - self.max_style_drop_rank)
            x0, x1 = self.q - 1, self.max_style_drop_rank - 1
            y0 = (np.exp((lvl - 0.5) * 2) - t0) / (centre - t0) * (1 - y00) + y00
            for xi in range(self.max_style_drop_rank, self.q):
                f[xi] = max((xi - x0) / (x1 - x0) * (1 - y0) + y0, 0)
        return f

    def __call__(self, x, lvl, R=None, s_out=None):
        if lvl == 0.5:
            return x
        require_cuda(x, "adjust_rank")
        fp16 = x.dtype == torch.float16
        xf = x.float().contiguous()
        f = torch.tensor(self.factors(lvl), dtype=torch.float32).to(x.device, non_blocking=True)
        out = ops.rank_adjust(xf, f, lvl < 0.5, _start(xf, self.q, R), niter=self.niter, s_out=s_out)
        return out.half() if fp16 else out
