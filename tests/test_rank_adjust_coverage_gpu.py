"""The image-context rank adjustment (vdb_rank_adjust_f32, lowrank.cu) element by element against the fp64 oracle, at every row
split, iteration count and spectrum it accepts, with all four outputs (out, s_out, u_out, v_out) checked directly.

Paths.  One 8-CTA cluster per item; CTA r holds rows [r cap, min(m, (r + 1) cap)) with cap = ceil(m / 8), so rank 7 holds
max(0, m - 7 cap) rows: none at m = 41 and 49 (it still joins every cluster barrier, Gram sum and all-gather), one at m = 57.
The launcher picks rank_adjust_kernel<4> when rw = ceil(cap / 8) <= 4 (m <= 256) and <5> above; m = 40 is the smallest tile
(5 rows per CTA) and m = 320 the largest (40 rows, the full shared-memory budget).  niter = 0 breaks out of the loop before any
Qm QR, so C = X qr(X^T R); niter 1, 2 and 7 leave the subspace unconverged, so a mis-ordered step shows.  Once the iteration
has converged, Y = X^T Qm has nearly orthogonal columns of graded norms, and CholeskyQR does not see column scaling, so even one
pass would be accurate there; only the first QR, of X^T R with mixed columns, sees the full condition of an exact-low-rank X
(~1e8), and at niter = 0 it is the last one, so the niter 0 rows at exact rank are what check the second pass.  The factor vectors
include a distinct value per index and one-hot vectors, so a slip in the eigenvalue order (perm) moves the result.  Every row of
CASES names the path it means to reach; the module asserts that the rows cover every m, niter, spectrum, factor kind and
keep_remainder value, and restates the launcher's rule for each m.

Yardsticks (u = 2^-24, fp32 unit roundoff; u64 = 2^-53).  The oracle runs torch.pca_lowrank's algorithm (Householder QR) on the
same fp32 x, R and fp32 factors, once in fp64 (the reference values) and once in fp32 (the reference's own rounding).
  out      |out - ref64| <= 4 e_ref + 1e-6 std(x) per element, e_ref = max |ref32 - ref64| (the merged yardstick of
           test_disentangle_gpu).  Both the oracle and the kernel compute the same subspace iteration from the same R; in exact
           arithmetic the QR's Q is unique up to column signs, which cancel in U diag(S f) V^T, so CholeskyQR2 and Householder
           differ only by rounding.  CholeskyQR2 in fp64 is backward stable while cond(Y) < u64^-1/2 ~ 1e8: the first pass
           leaves Q1 orthonormal to u64 cond(Y)^2, the second repairs it, and the result is rounded to fp32 (u per element), as
           Householder in fp32 ends.  At exact low rank r < 20 the fp32 X (rounded x, rounded centring) has 20 - r directions at
           the fp32 noise floor, cond(Y) ~ 1e7 < 1e8, so the Cholesky pivots stay positive; both the fp32 oracle and the kernel
           keep arbitrary noise directions there whose weight is at the fp32 floor of the products, which e_ref measures.
  L        the sign-free product L = U diag(S) V^T.  With E_L = ||L32 - L64||_2 (the fp32 oracle's first-order error), the kernel's
           ||L - L64||_2 <= 4 E_L + 3 u sum S: rounding u, s and v to fp32 moves each term sigma_k u_k v_k^T by at most 3 u sigma_k.
  s_out    descending, and per k  |s_k - S_k| <= dL + 3 u sum s + 10 u s_k + min(sqrt(m u64) s_1, m u64 s_1^2 / (2 s_k)),
           dL = ||L - L64||_2 measured.  s_k = sqrt(lambda_k) of the fp64 Gram of the kernel's fp32 C, i.e. sigma_k(C) up to the
           Gram's m u64 lambda_1 rounding (last term) and sigma_k(C Qn^T) up to Qn's orthonormality (<= 9 u, below); C Qn^T is
           the kernel's L before the output rounding (3 u sum s), and Weyl bounds |sigma_k(L) - S_k| by dL.
  U, V     columns up to sign where sigma_k is separated: with gap_k = min(min_{j != k} |S_k - S_j|, S_k) (the rank-20 L64's other
           singular values are those 19 and zeros) and gap_k > 4 dL, Wedin gives sin theta_k <= sqrt(2) dL / (gap_k - dL) for the
           singular vectors of the kernel's L, and ||a - b|| = 2 sin(theta / 2) <= sqrt(2) sin theta for unit vectors a, b:
           ||u_k -+ U_k|| <= 2 dL / (gap_k - dL) + 2 e_o + 2 u, e_o the measured orthonormality loss of the column pair.
  V^T V    |V^T V - I| <= 16 u: Qn leaves CholeskyQR2 orthonormal in fp64 and is rounded to fp32 (||dQn||_F <= sqrt(20) u, so
           ||Qn^T Qn - I||_2 <= 2 sqrt(20) u ~ 9 u), V = Qn Ub is formed in fp64 and rounded once more (2 u).
  U^T U    |U^T U - I|_jk <= 4 u + 1e-14 + (m + 64) u64 s_1^2 / (s_j s_k): u_k = C ub_k / s_k from the same fp32 C whose fp64 Gram
           the Jacobi solve diagonalised, so only the Gram's rounding (m u64 lambda_1), the eigenvectors' (<= 40 u64 lambda_1, plus
           the 1e-15 relative Jacobi threshold) and the two output roundings remain.  The bound grows as s_1 / s_k.
  std      std(out) = std(x) (unbiased, over the m * 768 elements of the item): out = fl(fl(x_new / a) b) with a = fl(std_new),
           b = fl(std_save), so |std(out) / std(x) - 1| <= 2 u (a, b) + 2 u rms(out) / std(out) (the two per-element roundings) +
           2 eps_std, eps_std = 256 u64 mean(y^2) / var(y) for the fp64 sums of at most ~200 terms in order.  That is below
           1 / (2 m 768), the std's change when the x side alone takes the biased count, on every row whose rows are not offset
           far from zero (rms / std ~ 1); the `offset` spectrum (rms / std ~ 1e3) is checked against its bound only.  A count
           that is wrong on both sides cancels in std(x) / std(x_new) and leaves out unchanged up to rounding, so no output can
           show it; the check catches a std whose count differs between the two sides.

Identities, with their own bounds (test docstrings): factors 1 with keep_remainder gives x; factors 0 without it gives rows
constant bit for bit; an item with X = 0 gives S = 0, zero U and V columns and x_remain = 0 as torch.pca_lowrank.  Bitwise:
x 2^k and -x (test_scaling_and_negation_are_exact), batches against single calls, an item of NaN against its neighbours, and
repeated calls.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
N, Q, CLUSTER, WARPS = 768, 20, 8, 8
U = 2.0 ** -24
U64 = 2.0 ** -53
SLACK = 1.0 + 2.0 ** -10
OUTLIER_COLS = (3, 100, 401, 402, 767)


# ---------------------------------------------------------------------------------------------------------------------------
# the launcher's row split and instantiation rule, restated
# ---------------------------------------------------------------------------------------------------------------------------
def rows_per_cta(m):
    return -(-m // CLUSTER)


def instantiation(m):
    """rank_adjust_kernel<RW> the launcher picks: rw = ceil(rows_cap / 8) warps' rows per CTA, <4> for rw <= 4, else <5>."""
    rw = -(-rows_per_cta(m) // WARPS)
    return 4 if rw <= 4 else 5


def last_cta_rows(m):
    cap = rows_per_cta(m)
    return max(0, min(m, CLUSTER * cap) - (CLUSTER - 1) * cap)


M_VALUES = (40, 41, 49, 57, 255, 256, 257, 300, 320)
assert {m: instantiation(m) for m in M_VALUES} == {40: 4, 41: 4, 49: 4, 57: 4, 255: 4, 256: 4, 257: 5, 300: 5, 320: 5}
assert {m: last_cta_rows(m) for m in M_VALUES} == {40: 5, 41: 0, 49: 0, 57: 1, 255: 31, 256: 32, 257: 26, 300: 34, 320: 40}
assert rows_per_cta(40) == 5 and rows_per_cta(320) == 40


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
SPECTRA = ("gauss", "gapped", "dominant", "outliers", "geometric", "neartie", "tie20", "rank1", "rank5", "rank19", "offset")


def _orth(rows, k, g, centre=False):
    a = torch.randn(rows, k, generator=g, dtype=torch.float64)
    if centre:
        a = a - a.mean(0, keepdim=True)       # columns orthogonal to the ones vector: the row centring keeps the spectrum
    return torch.linalg.qr(a).Q


def _with_spectrum(m, sigma, g):
    """U diag(sigma) V^T with V's columns orthogonal to the ones vector (so X has exactly this spectrum), plus a per-row offset
    that the centring removes."""
    sigma = torch.as_tensor(sigma, dtype=torch.float64)
    x = (_orth(m, len(sigma), g) * sigma) @ _orth(N, len(sigma), g, centre=True).T
    return x + 0.1 * sigma[0] / math.sqrt(N) * torch.randn(m, 1, generator=g, dtype=torch.float64)


def spectrum_input(spec, m, seed=0):
    """x [1, m, 768] fp32 with the named spectrum of its row-centred X."""
    g = torch.Generator().manual_seed(1000 * seed + 7 * m + SPECTRA.index(spec))
    k = torch.arange(m, dtype=torch.float64)
    tail = lambda top, n: top * torch.linspace(1.0, 0.5, n, dtype=torch.float64)
    if spec == "gauss":
        x = torch.randn(m, N, generator=g, dtype=torch.float64)
    elif spec == "gapped":                    # the golden's gapped input at any m: singular values 30 .. 11 over noise 0.02
        u, v = _orth(m, Q, g), _orth(N, Q, g)
        x = (u * torch.linspace(30.0, 11.0, Q, dtype=torch.float64)) @ v.T + 0.02 * torch.randn(m, N, generator=g, dtype=torch.float64) + 0.05
    elif spec == "dominant":                  # sigma_1 / sigma_2 = 1e3
        x = _with_spectrum(m, torch.cat([torch.tensor([1e3], dtype=torch.float64), tail(1.0, m - 1)]), g)
    elif spec == "outliers":                  # CLIP-like feature columns 50x the rest
        x = torch.randn(m, N, generator=g, dtype=torch.float64)
        x[:, list(OUTLIER_COLS)] *= 50.0
    elif spec == "geometric":                 # sigma_k = 10^(-k/4) over the kept 20, then a flat tail at half sigma_20
        x = _with_spectrum(m, torch.cat([10.0 ** (-k[:Q] / 4), tail(0.5 * 10.0 ** (-(Q - 1) / 4), m - Q)]), g)
    elif spec == "neartie":                   # pairs with relative gap 1e-4
        top = 10.0 * 0.8 ** (k[:Q] // 2)
        top[1::2] *= 1.0 - 1e-4
        x = _with_spectrum(m, torch.cat([top, tail(0.5 * top[-1].item(), m - Q)]), g)
    elif spec == "tie20":                     # sigma_20 = sigma_21: the tie straddles the kept rank
        top = torch.linspace(10.0, 2.0, Q, dtype=torch.float64)
        x = _with_spectrum(m, torch.cat([top, top[-1:], tail(1.0, m - Q - 1)]), g)
    elif spec.startswith("rank"):             # exact rank r < 20
        r = int(spec[4:])
        x = _with_spectrum(m, torch.linspace(10.0, 5.0, r, dtype=torch.float64), g)
    elif spec == "offset":                    # rows at 1e3 with a spread of 1
        x = 1e3 + torch.randn(m, N, generator=g, dtype=torch.float64)
    else:
        raise ValueError(spec)
    return x.float()[None]


def start(m, seed=5):
    return torch.randn(m, Q, generator=torch.Generator().manual_seed(seed))


FACTORS = ("lvl0.1", "lvl0.25", "lvl0.75", "lvl0.9", "random", "ones", "zeros", "onehot0", "onehot10", "onehot19")


def factors(name):
    """fp32-representable fp64 [20]: the kernel's and both oracles' factors are the same numbers."""
    if name.startswith("lvl"):
        from lib.model_zoo.disentangle import adjust_rank
        f = adjust_rank().factors(float(name[3:]))
    elif name == "random":
        f = np.random.default_rng(7).uniform(0.0, 2.0, Q)
        assert len(set(f.astype(np.float32).tolist())) == Q
    elif name == "ones":
        f = np.ones(Q)
    elif name == "zeros":
        f = np.zeros(Q)
    elif name.startswith("onehot"):
        f = np.zeros(Q)
        f[int(name[6:])] = 1.0
    return f.astype(np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------------------
def _case(m, niter, spec, fac, keep, path):
    return dict(id=f"m{m}-n{niter}-{spec}-{fac}-{'keep' if keep else 'drop'}", m=m, niter=niter, spec=spec, fac=fac, keep=keep,
                path=path)


CASES = [
    _case(40, 100, "gauss", "lvl0.25", True, "<4>, smallest tile: 5 rows in every CTA"),
    _case(40, 7, "geometric", "random", False, "<4>, smallest tile; CholeskyQR2 at cond(X^T R) ~ 1e5"),
    _case(40, 2, "tie20", "onehot19", True, "<4>, smallest tile; the tie across the kept rank, weighted alone"),
    _case(41, 100, "gauss", "lvl0.9", False, "rank 7 holds no rows"),
    _case(41, 1, "rank1", "onehot0", True, "rank 7 holds no rows; exact rank 1"),
    _case(41, 100, "rank19", "random", False, "rank 7 holds no rows; exact rank 19, one noise direction kept"),
    _case(41, 0, "rank5", "lvl0.75", False, "rank 7 holds no rows; niter 0 at exact rank 5: Qn is CholeskyQR2 of an X^T R of "
          "condition ~1e8 whose columns are not graded, where one pass would leave Qn orthonormal to ~1e-1 only"),
    _case(49, 0, "dominant", "onehot0", True, "rank 7 holds no rows; niter 0 (no Qm QR)"),
    _case(49, 100, "rank5", "random", False, "rank 7 holds no rows; exact rank 5"),
    _case(49, 7, "neartie", "onehot10", True, "rank 7 holds no rows; near-tied pairs"),
    _case(57, 0, "outliers", "lvl0.1", True, "rank 7 holds one row; niter 0"),
    _case(57, 100, "neartie", "onehot10", False, "rank 7 holds one row; near-tied pairs"),
    _case(57, 2, "offset", "random", True, "rank 7 holds one row; rows far from zero"),
    _case(255, 0, "gauss", "random", False, "<4> below the boundary; niter 0"),
    _case(255, 100, "tie20", "onehot19", True, "<4>; the tie across the kept rank"),
    _case(256, 100, "gapped", "lvl0.75", False, "<4> at the boundary; the golden's gapped spectrum"),
    _case(256, 100, "geometric", "random", True, "<4> at the boundary; steep decay"),
    _case(256, 7, "rank19", "zeros", True, "<4>; exact rank 19, all factors 0 (x minus its rank-20 part)"),
    _case(256, 2, "offset", "lvl0.25", True, "<4>; rows far from zero"),
    _case(257, 1, "gauss", "random", True, "<5> at the boundary; niter 1"),
    _case(257, 100, "rank1", "onehot0", True, "<5>; exact rank 1"),
    _case(257, 0, "rank1", "random", True, "<5>; niter 0 at exact rank 1: the first CholeskyQR2 is the last"),
    _case(257, 7, "dominant", "lvl0.1", False, "<5>; one dominant direction"),
    _case(300, 2, "neartie", "lvl0.9", False, "<5>; near-tied pairs, unconverged"),
    _case(300, 100, "dominant", "random", False, "<5>; one dominant direction"),
    _case(300, 100, "outliers", "onehot19", False, "<5>; outlier feature columns"),
    _case(300, 1, "gapped", "onehot0", True, "<5>; niter 1"),
    _case(320, 0, "gapped", "ones", False, "<5>, largest tile: 40 rows in every CTA; niter 0"),
    _case(320, 100, "geometric", "onehot10", True, "<5>, largest tile; steep decay"),
    _case(320, 7, "offset", "random", False, "<5>, largest tile; rows far from zero"),
    _case(320, 1, "rank5", "lvl0.1", True, "<5>, largest tile; exact rank 5"),
    _case(320, 100, "rank19", "lvl0.75", True, "<5>, largest tile; exact rank 19"),
]
assert {c["m"] for c in CASES} == set(M_VALUES)
assert {c["niter"] for c in CASES} == {0, 1, 2, 7, 100}
assert {c["spec"] for c in CASES} == set(SPECTRA)
assert {c["fac"] for c in CASES} == set(FACTORS)
assert {c["keep"] for c in CASES} == {True, False}
assert len({c["id"] for c in CASES}) == len(CASES)
assert {instantiation(c["m"]) for c in CASES} == {4, 5} and any(last_cta_rows(c["m"]) == 0 for c in CASES)


# ---------------------------------------------------------------------------------------------------------------------------
# running the kernel and the oracle
# ---------------------------------------------------------------------------------------------------------------------------
def run(x, R, f, keep, niter, outputs=True):
    """-> (out, s, u, v) on the CPU; the optional outputs start as NaN so an element the kernel does not write shows."""
    from vdb200 import ops
    n, m, _ = x.shape
    nan = float("nan")
    s = torch.full((n, Q), nan, device=DEV) if outputs else None
    u = torch.full((n, m, Q), nan, device=DEV) if outputs else None
    v = torch.full((n, N, Q), nan, device=DEV) if outputs else None
    out = ops.rank_adjust(x.to(DEV).contiguous(), torch.as_tensor(f, dtype=torch.float32, device=DEV), keep, R.to(DEV), niter=niter,
                          s_out=s, u_out=u, v_out=v)
    torch.cuda.synchronize()
    if not outputs:
        return out.cpu()
    return out.cpu(), s.cpu(), u.cpu(), v.cpu()


def oracle(x, R, f, keep, niter):
    from oracle.disentangle_oracle import rank_adjust_factors
    ref64, U64_, S64, V64 = rank_adjust_factors(x, R, f, keep, niter, torch.float64)
    ref32, U32_, S32, V32 = rank_adjust_factors(x, R, f.astype(np.float32), keep, niter, torch.float32)
    return (ref64, U64_[0], S64[0], V64[0]), (ref32.double(), U32_[0].double(), S32[0].double(), V32[0].double())


def product(u, s, v):
    return (u * s) @ v.T


def spec_norm(a):
    return torch.linalg.matrix_norm(a, ord=2).item()


def std_eps(y):
    """fp64 relative error bound of the kernel's one-pass (sum, sum of squares) std: 256 u64 mean(y^2) / var(y)."""
    y = y.double()
    return 256 * U64 * (y * y).mean().item() / y.var().item()


def std_bound(x, out):
    """|std(out) / std(x) - 1| bound of the module docstring."""
    o = out.double()
    return (2 * U + 2 * U * (o * o).mean().sqrt().item() / o.std().item() + 2 * std_eps(x) + 2 * std_eps(out)) * SLACK


# ---------------------------------------------------------------------------------------------------------------------------
# the case table: out, s_out, u_out, v_out and std against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_case(case):
    m, niter, keep = case["m"], case["niter"], case["keep"]
    x = spectrum_input(case["spec"], m)
    R = start(m)
    f = factors(case["fac"])
    (ref64, U64_, S64, V64), (ref32, U32_, S32, V32) = oracle(x, R, f, keep, niter)
    out, s, u, v = run(x, R, f, keep, niter)
    s, u, v = s[0].double(), u[0].double(), v[0].double()
    tag = f"{case['id']} (<{instantiation(m)}>, rank 7 holds {last_cta_rows(m)} rows: {case['path']})"

    # out per element
    e_ref = (ref32 - ref64).abs().max().item()
    e_out = (out.double() - ref64).abs().max().item()
    tol = 4 * e_ref + 1e-6 * x.double().std().item()
    print(f"{tag}\n  out {e_out:.3g} / bound {tol:.3g} (fp32 reference {e_ref:.3g})")
    assert e_out <= tol, (case["id"], e_out, e_ref)

    # the optional outputs are written and do not change out
    assert torch.isfinite(s).all() and torch.isfinite(u).all() and torch.isfinite(v).all(), case["id"]
    assert torch.equal(run(x, R, f, keep, niter, outputs=False), out), case["id"]

    # the sign-free product U diag(S) V^T
    L64 = product(U64_, S64, V64)
    E_L = spec_norm(product(U32_, S32, V32) - L64)
    dL = spec_norm(product(u, s, v) - L64)
    tol_L = 4 * E_L + 3 * U * S64.sum().item()
    print(f"  ||L - L64||_2 {dL:.3g} / bound {tol_L:.3g} (fp32 reference {E_L:.3g})")
    assert dL <= tol_L, (case["id"], dL, E_L)

    # s_out: descending, and against S64
    assert (s[:-1] >= s[1:]).all(), (case["id"], s)
    s1 = s[0].item()
    tol_s = (dL + 3 * U * s.sum().item() + 10 * U * s +
             torch.minimum(torch.full_like(s, math.sqrt(m * U64) * s1), m * U64 * s1 ** 2 / (2 * s.clamp_min(1e-300)))) * SLACK
    err_s = (s - S64).abs()
    print(f"  s: max |s - S| / bound {(err_s / tol_s).max().item():.3g}, max relative {(err_s / S64.clamp_min(1e-300)).max().item():.3g}")
    assert (err_s <= tol_s).all(), (case["id"], err_s, tol_s)

    # orthonormality in fp64
    ev = (v.T @ v - torch.eye(Q, dtype=torch.float64)).abs()
    print(f"  |V^T V - I| {ev.max().item() / U:.3g} u / 16 u")
    assert ev.max().item() <= 16 * U, (case["id"], ev.max().item())
    sj = s.clamp_min(1e-300)
    tol_u = 4 * U + 1e-14 + (m + 64) * U64 * s1 ** 2 / (sj[:, None] * sj[None, :])
    eu = (u.T @ u - torch.eye(Q, dtype=torch.float64)).abs()
    print(f"  |U^T U - I| / bound {(eu / tol_u).max().item():.3g}")
    assert (eu <= tol_u).all(), (case["id"], (eu / tol_u).max().item())

    # separated columns of U and V, up to sign
    checked = []
    for k in range(Q):
        others = torch.cat([S64[:k], S64[k + 1:]])
        gap = min((others - S64[k]).abs().min().item(), S64[k].item())
        if gap <= 4 * dL:
            continue
        sign = 1.0 if (u[:, k] @ U64_[:, k]).item() >= 0 else -1.0
        e_o = max(eu[k].max().item(), ev[k].max().item())
        tol_c = 2 * dL / (gap - dL) + 2 * e_o + 2 * U
        eu_k = (u[:, k] - sign * U64_[:, k]).norm().item()
        ev_k = (v[:, k] - sign * V64[:, k]).norm().item()
        assert eu_k <= tol_c and ev_k <= tol_c, (case["id"], k, eu_k, ev_k, tol_c)
        checked.append(k)
    print(f"  columns checked up to sign: {checked}")

    # std(out) = std(x), unbiased
    rel = abs(out.double().std().item() / x.double().std().item() - 1.0)
    tol_std = std_bound(x, out)
    biased = 1.0 / (2 * m * N)
    print(f"  std: {rel:.3g} / bound {tol_std:.3g} (a biased count on one side moves it by {biased:.3g})")
    assert rel <= tol_std, (case["id"], rel, tol_std)
    if case["spec"] != "offset":
        assert tol_std < biased / 2, (case["id"], tol_std)


# ---------------------------------------------------------------------------------------------------------------------------
# identities
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,spec,niter", [(41, "gauss", 100), (257, "rank5", 2), (320, "outliers", 0), (57, "offset", 7)])
def test_unit_factors_with_remainder_return_x(m, spec, niter):
    """factors = 1 with keep_remainder: out = x + C (W - I) Qn^T with W - I at the fp64 eigenvector error (|d| <= 1e-12 S_1 per
    element), so only the fp32 centring and the std ratio remain.  With mu = fl(mean) (within u |mean|), x_new = fl(fl(x - mu) +
    mu) + d errs by e = u (|x - mean| + |x| + |mean|) + |d| (each fl one u of its result).  std(x_new) / std(x) is within
    sqrt(N / (N - 1)) rms(e) / std(x) (Minkowski) and the two fp64 std's within eps_std each, so with a = fl(std_new),
    b = fl(std_save) the ratio r = b / a is within rho = sqrt(N / (N - 1)) rms(e) / std(x) + 2 eps_std + 2 u of 1, and
    out = fl(fl(x_new / a) b):   |out - x| <= e + (rho + 2 u) (|x| + e)."""
    x = spectrum_input(spec, m)
    R = start(m)
    out, s, _, _ = run(x, R, np.ones(Q), True, niter)
    xd = x.double()[0]
    mean = xd.mean(-1, keepdim=True)
    e = U * ((xd - mean).abs() + xd.abs() + mean.abs()) * SLACK + 1e-12 * s[0, 0].item()
    cnt = m * N
    rho = math.sqrt(cnt / (cnt - 1)) * e.pow(2).mean().sqrt().item() / xd.std().item() + 2 * std_eps(x) + 2 * U
    tol = e + (rho + 2 * U) * (xd.abs() + e) * SLACK
    err = (out[0].double() - xd).abs()
    print(f"m {m} {spec} niter {niter}: max |out - x| / bound {(err / tol).max().item():.3g}, max |out - x| {err.max().item():.3g}")
    assert (err <= tol).all(), (err / tol).max().item()


@pytest.mark.parametrize("m,spec,niter", [(49, "gauss", 1), (256, "gapped", 100), (300, "dominant", 7)])
def test_zero_factors_without_remainder_give_constant_rows(m, spec, niter):
    """factors = 0 without keep_remainder: W = 0 exactly (every product has a factor 0), so C W = 0, d = 0 and x_new = mu, each
    row's fp32 mean: every row of out is one value, bit for bit.  That value is mean_i std(x) / std(means) (the std of the
    m x 768 matrix of row means): mu = mean (1 + u), std(mu) is within r_mu = sqrt(N / (N - 1)) rms(mu - mean) / std(means) <=
    1.001 u rms(means) / std(means) of std(means), the fp64 std's within eps_std, and fl(std), fl(x_new / a) and fl(. b) add
    one u each:   |out_i / ref_i - 1| <= 5 u + r_mu + 2 eps_std."""
    x = spectrum_input(spec, m)
    R = start(m)
    out, s, u, v = run(x, R, np.zeros(Q), False, niter)
    o = out[0]
    assert torch.equal(o, o[:, :1].expand_as(o)), "rows not constant"
    xd = x.double()[0]
    means = xd.mean(-1, keepdim=True)
    mm = means.expand_as(xd)
    ref = means[:, 0] * xd.std() / mm.std()
    r_mu = 1.001 * U * mm.pow(2).mean().sqrt().item() / mm.std().item()
    tol = (5 * U + r_mu + 2 * std_eps(x) + 2 * std_eps(mm)) * SLACK
    rel = ((o[:, 0].double() - ref).abs() / ref.abs()).max().item()
    print(f"m {m} {spec}: max relative {rel:.3g} / bound {tol:.3g}")
    assert rel <= tol


def test_item_with_zero_centred_rows():
    """Rows that are each constant (values with <= 14 significant bits, so every partial row sum is exact and X = 0 exactly, on
    the device and in torch): the Cholesky pivots take the 1e-300 clamp on a zero Gram, Qn = 0, C = 0 and the Jacobi matrix is
    0.  S = 0, u_out and v_out are zero (U = X V / S is undefined, and vdb200.h defines it as 0), so decompose's
    x_remain = X - U diag(S) V^T = 0, as torch.pca_lowrank's finite U, S = 0 give in the oracle.  out = x_new / std(x_new)
    std(x) with x_new = mu = x exactly, both std's of the same values in different orders: |out - ref| <= (4 u + 2 eps_std) |ref|,
    with or without the remainder and for any factors."""
    from lib.model_zoo.disentangle import decompose
    from oracle.disentangle_oracle import lowrank, rank_adjust_factors
    m = 41
    c = torch.round(torch.randn(1, m, 1, generator=torch.Generator().manual_seed(2)) * 64) / 64
    x = c.expand(1, m, N).contiguous()
    R = start(m)
    for keep, fac in ((True, "random"), (False, "lvl0.25"), (False, "zeros")):
        f = factors(fac)
        out, s, u, v = run(x, R, f, keep, 3)
        ref, _, S64, _ = rank_adjust_factors(x, R, f, keep, 3)
        assert torch.equal(s, torch.zeros_like(s)) and (S64 == 0).all()
        assert torch.equal(u, torch.zeros_like(u)), "u_out of a zero singular value must be 0"
        assert torch.equal(v, torch.zeros_like(v))
        tol = (4 * U + 2 * std_eps(x)) * SLACK
        rel = ((out.double() - ref).abs() / ref.abs().clamp_min(1e-300)).max().item()
        assert rel <= tol, (keep, fac, rel, tol)
    U_, s_, v_, x_mean, x_remain = decompose(x.to(DEV), R=R.to(DEV), niter=3)
    Uo, So, Vo = lowrank(x.double() - x.double().mean(-1, keepdim=True), R.double(), 3)
    remain64 = (x.double() - x.double().mean(-1, keepdim=True)) - torch.bmm(Uo * So[:, None, :], Vo.transpose(1, 2))
    assert torch.isfinite(Uo).all() and (remain64 == 0).all()
    assert torch.equal(x_remain.cpu(), torch.zeros_like(x)), "decompose's x_remain of X = 0 must be 0"


# ---------------------------------------------------------------------------------------------------------------------------
# bitwise metamorphic checks
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,spec,keep", [(41, "gauss", True), (257, "gapped", False)])
def test_scaling_and_negation_are_exact(m, spec, keep):
    """x 2^k -> out 2^k, s 2^k, u and v unchanged; -x -> -out, s, u, -v; bit for bit.  Every step commutes with an exact power of
    two or a sign: fp32 / fp64 products, sums and the row mean scale exactly, sqrt of a value times 2^(2k) is sqrt times 2^k, the
    quotients (L^-1, acc / sqrt(lambda), x_new / std_new) are correctly rounded ratios of scaled operands, and the Jacobi test
    |a_pq| > 1e-15 sqrt(|a_pp a_qq|) and the 1e150 cut on theta are scale-free; negating X negates Y = X^T R, Qn and V, keeps
    C = X Qn (two signs), its Gram, W and U, and negates d and x_new.  Nothing leaves the normal range: for these full-rank
    inputs at k = -40 the smallest Gram pivot is ~(2^-40 sigma_min(Y))^2 ~ 1e-20, far above the 1e-300 clamp, the smallest
    fp32 intermediates (~1e-20) far above 1.2e-38, and at k = 40 the largest (|x| ~ 2^43, Gram ~ 1e33) far below the limits."""
    x = spectrum_input(spec, m)
    R = start(m)
    f = factors("random")
    base = run(x, R, f, keep, 7)
    for k in (-40, -12, 12, 40):
        sc = 2.0 ** k
        out, s, u, v = run(x * sc, R, f, keep, 7)
        assert torch.equal(out, base[0] * sc) and torch.equal(s, base[1] * sc), k
        assert torch.equal(u, base[2]) and torch.equal(v, base[3]), k
    out, s, u, v = run(-x, R, f, keep, 7)
    assert torch.equal(out, -base[0]) and torch.equal(s, base[1]) and torch.equal(u, base[2]) and torch.equal(v, -base[3])


# ---------------------------------------------------------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------------------------------------------------------
def _batch(m, n):
    """n items of different spectra and scales 10^-2 .. 10^2."""
    return torch.cat([spectrum_input(SPECTRA[i % len(SPECTRA)], m, seed=i) * 10.0 ** ((i % 9 - 4) / 2) for i in range(n)])


@pytest.mark.parametrize("m", [49, 300])
def test_batch_of_40_equals_single_calls(m):
    """40 items need several waves of 8-CTA clusters on 132 SMs (at most 16 resident at once); each item's cluster computes the
    same fixed-order reductions as a single call, so every output equals the single call bit for bit.  Two identical calls are
    equal, and an item of NaN leaves every other item unchanged."""
    n = 40
    x = _batch(m, n)
    R = start(m)
    f = factors("random")
    out, s, u, v = run(x, R, f, False, 100)
    for i in range(n):
        oi, si, ui, vi = run(x[i:i + 1], R, f, False, 100)
        assert torch.equal(out[i:i + 1], oi) and torch.equal(s[i:i + 1], si), i
        assert torch.equal(u[i:i + 1], ui) and torch.equal(v[i:i + 1], vi), i
    again = run(x, R, f, False, 100)
    assert all(torch.equal(a, b) for a, b in zip(again, (out, s, u, v)))
    bad = x.clone()
    bad[7, 3, 11] = float("nan")
    nout, ns, nu, nv = run(bad, R, f, False, 100)
    keep = [i for i in range(n) if i != 7]
    assert torch.equal(nout[keep], out[keep]) and torch.equal(ns[keep], s[keep])
    assert torch.equal(nu[keep], u[keep]) and torch.equal(nv[keep], v[keep])
    assert torch.isnan(nout[7]).any()


# ---------------------------------------------------------------------------------------------------------------------------
# the wrapper's refusals
# ---------------------------------------------------------------------------------------------------------------------------
def test_out_of_another_shape_or_overlapping_x_is_refused():
    """A short out would be written past its end, and an out that overlaps x breaks the kernel's no-alias contract (a shifted
    one writes rows another item's cluster has yet to read): both are ValueErrors before any launch."""
    from vdb200 import ops
    m = 256
    buf = torch.randn(3 * m * N, device=DEV)
    x = buf[:2 * m * N].view(2, m, N)
    f = torch.ones(Q, device=DEV)
    R = start(m).to(DEV)
    bad = {
        "short": torch.empty(2, m - 1, N, device=DEV),
        "one item": torch.empty(1, m, N, device=DEV),
        "flat": torch.empty(2 * m * N, device=DEV),
        "x itself": x,
        "shifted one item": buf[m * N:].view(2, m, N),
        "shifted one row": buf[N:N + 2 * m * N].view(2, m, N),
    }
    for name, out in bad.items():
        ops.reset_launch_count()
        with pytest.raises(ValueError, match="rank_adjust: out"):
            ops.rank_adjust(x, f, True, R, out=out)
        assert ops.launch_count() == 0, name
    ops.reset_launch_count()
    ops.rank_adjust(x, f, True, R, out=buf.new_empty(2, m, N))
    assert ops.launch_count() == 1
