"""Reference restatement of app.py's decompose + adjust_rank (app.py:48-127) with the Gaussian start R injected.

Same algorithm and the same torch ops as torch.pca_lowrank(center=False) on the row-centred tokens (Householder QR through
torch.linalg.qr, torch.linalg.svd on the q x m matrix B), batched over items as the reference batches them, in fp32 (what the
reference computes) or fp64 (the accuracy yardstick).  One difference from the reference: each item is rescaled by its own
standard deviation (the reference broadcasts the [n] std vector against the feature axis, which only runs for n = 1).
"""
import hashlib

import torch


def golden_inputs():
    """The two [1, 256, 768] inputs of tests/golden/disentangle.npz, regenerated from their seed (the fixture keeps their SHA-256,
    not the 1.5 MB of values): a standard Gaussian, and a matrix with a spectral gap after the 20th singular value (20 directions
    of singular values 30 .. 11 over Gaussian noise of std 0.02, about 0.15 overall).  Rounded to fp16-representable fp32 values,
    so a last-bit difference in the CPU's libm or LAPACK does not change them."""
    g = torch.Generator().manual_seed(31)
    gauss = torch.randn(1, 256, 768, generator=g)
    u = torch.linalg.qr(torch.randn(256, 20, generator=g, dtype=torch.float64)).Q
    v = torch.linalg.qr(torch.randn(768, 20, generator=g, dtype=torch.float64)).Q
    s = torch.linspace(30.0, 11.0, 20, dtype=torch.float64)
    gap = (u * s) @ v.T + 0.02 * torch.randn(256, 768, generator=g, dtype=torch.float64) + 0.05
    return [t.half().float() for t in (gauss, gap.float()[None])]


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def lowrank(X, R, niter):
    """torch._lowrank._svd_lowrank for m < n with R given: (U [n,m,q], S [n,q], V [n,d,q]) of X [n, m, d] (d > m)."""
    A = X.mH                                   # [n, d, m]
    Q = torch.linalg.qr(torch.matmul(A, R)).Q
    for _ in range(niter):
        Q = torch.linalg.qr(torch.matmul(A.mH, Q)).Q
        Q = torch.linalg.qr(torch.matmul(A, Q)).Q
    B = torch.matmul(Q.mH, A)
    Ub, S, Vh = torch.linalg.svd(B, full_matrices=False)
    return Vh.mH, S, Q.matmul(Ub)


def rank_adjust(x, R, factors, keep_remainder, niter=100, dtype=torch.float64):
    """x [n, m, d] -> (x_new, S before scaling) in `dtype`; factors [q] scale S (app.py's s[:, xi] *= yi)."""
    x = x.to(dtype)
    R = R.to(dtype)
    std_save = x.std(dim=(-2, -1), keepdim=True)
    x_mean = x.mean(-1, keepdim=True)
    X = x - x_mean
    U, S, V = lowrank(X, R, niter)
    x_lowrank = torch.bmm(torch.bmm(U, torch.diag_embed(S)), V.permute(0, 2, 1))
    x_remain = X - x_lowrank if keep_remainder else 0
    Sf = S * torch.as_tensor(factors, dtype=dtype, device=x.device)
    x_new = torch.bmm(torch.bmm(U, torch.diag_embed(Sf)), V.permute(0, 2, 1)) + x_mean + x_remain
    x_new = x_new / x_new.std(dim=(-2, -1), keepdim=True) * std_save
    return x_new, S
