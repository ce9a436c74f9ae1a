"""Stochastic DPM-Solver++ (DPMSolverSDESampler), CPU side: the table at eta = 0 is the ODE table bit for bit; at eta > 0 its rows
fold the fp64 direct SDE step (oracle/dpm_sde_oracle.py); the last row is deterministic; the sampler's argument checks; the refusals
of vdb_dpmpp_sde_cfg_step; weak convergence of the oracle's SDE walk on the analytic Gaussian model."""
import types

import numpy as np
import pytest
import torch

from oracle import dpm_sde_oracle as G
from oracle import dpm_solver_oracle as D
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]


def _ts(grid, steps, walk=None):
    return G.grid(grid, steps, AC.numpy())[:walk]


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("grid", ["uniform", "trailing", "karras"])
def test_eta_zero_is_the_ode_table_bit_for_bit(order, grid):
    from lib.model_zoo.dpm_solver import dpmpp_table
    for steps, walk in ((5, None), (14, None), (20, None), (50, None), (50, 12), (100, None)):
        ts = _ts(grid, steps, walk)
        ode = dpmpp_table(AC, ts, order)
        sde = dpmpp_table(AC, ts, order, eta=0.0)
        assert ode.tobytes() == sde.tobytes(), (grid, steps, walk)
        assert ode.tobytes() == dpmpp_table(AC, ts, order, 0).tobytes()
        assert not ode[:, 6:].any()


def _oracle_row(ts, order, eta, i):
    """Coefficients of x, x0_i, x0_{i+1}, x0_{i+2} and z in the oracle's step at grid index i, read off its direct step on unit
    inputs (the step is linear in them): eps is chosen so that the data predictions take prescribed values, the state entering
    step i is set by `after`, and z is 1 at step i alone."""
    alpha, sigma = D.coefficients(AC.numpy(), ts)[:2]
    n = len(ts)
    coefs = []
    for lane in range(5):                                   # x, x0_i, x0_{i+1}, x0_{i+2}, z
        x_in = 1.0 if lane == 0 else 0.0
        x0_at = {i: float(lane == 1), i + 1: float(lane == 2), i + 2: float(lane == 3)}
        trace = []
        G.walk(np.array(x_in if i == n - 1 else 0.0), lambda x, j: (x - alpha[j] * x0_at.get(j, 0.0)) / sigma[j], AC.numpy(),
               ts, order, eta=eta, noise=lambda j: np.array(float(lane == 4 and j == i)), trace=trace,
               after=lambda j, xn: np.array(x_in) if j == i + 1 else xn)
        coefs.append(trace[n - 1 - i][2])
    return np.array(coefs, dtype=np.float64)


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("eta", [0.5, 1.0])
@pytest.mark.parametrize("grid,steps,walk", [("uniform", 20, None), ("karras", 20, None), ("trailing", 14, None),
                                             ("karras", 50, 12)])
def test_sde_rows_fold_the_oracle_step(order, eta, grid, steps, walk):
    from lib.model_zoo.dpm_solver import dpmpp_table
    ts = _ts(grid, steps, walk)
    table = dpmpp_table(AC, ts, order, eta)
    assert table.shape == (len(ts), 8) and not table[:, 7].any()
    alpha, sigma = D.coefficients(AC.numpy(), ts)[:2]
    for i in range(len(ts)):
        P, Q, A, B, C, Dd, N = table[i, :7]
        assert P == 1.0 / alpha[i] and Q == -sigma[i] / alpha[i]
        got = np.array([A, B, C, Dd, N])
        want = _oracle_row(ts, order, eta, i)
        assert np.allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max()), (i, got, want)
    assert table[0, 6] == 0.0, "the last step is deterministic"
    assert (table[1:, 6] > 0).all()


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def test_sampler_argument_checks():
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler, dpmpp_table
    for bad in (0, 4, "2"):
        with pytest.raises(ValueError, match="order"):
            DPMSolverSDESampler(_fake_model(), order=bad)
    S = DPMSolverSDESampler(_fake_model(), order=3, grid="karras")
    assert isinstance(S, DPMSolverSampler) and S.order == 3 and S.eta == 1.0
    c = {"type": "text", "conditioning": torch.zeros(1, 77, 768), "unconditional_conditioning": torch.zeros(1, 77, 768),
         "unconditional_guidance_scale": 7.5}
    state = torch.get_rng_state()
    for bad in (-0.1, 1.5, float("nan"), float("inf"), -float("inf"), "x", None, [0.5]):
        with pytest.raises(ValueError, match="eta"):
            S.sample(steps=10, shape=[1, 4, 8, 8], x_info={"type": "image"}, c_info=c, eta=bad, verbose=False)
        with pytest.raises(ValueError, match="eta"):
            S.sample_multicontext(steps=10, shape=[1, 4, 8, 8], x_info={"type": "image"}, c_info_list=[c], eta=bad, verbose=False)
    assert torch.equal(torch.get_rng_state(), state), "a refused call draws nothing"
    with pytest.raises(ValueError, match="ddim_eta"):
        S.make_schedule(10, ddim_eta=0.5, verbose=False)
    for m in ("p_sample_ddim", "invert"):
        with pytest.raises(NotImplementedError):
            getattr(S, m)({"x": None}, c, None, 0)
    with pytest.raises(NotImplementedError):
        S.p_sample_ddim_multicontext({"x": None}, [c], None, 0)
    with pytest.raises(NotImplementedError):
        S.invert_multicontext(10, None, [c])
    # the CPU model stops the walk after the modes are built: the key is drawn only at eta > 0
    for eta, draws in ((0.0, False), (0.3, True), (1, True)):
        torch.manual_seed(0)
        before = torch.get_rng_state()
        with pytest.raises(RuntimeError, match="CPU"):
            S.sample(steps=10, shape=[1, 4, 8, 8], x_info={"type": "image"}, c_info=c, eta=eta, verbose=False)
        assert torch.equal(torch.get_rng_state(), before) != draws, eta
        assert S.eta == float(eta)
    S.make_schedule(20, verbose=False)
    S.eta = 0.7
    assert S._graph_tag() == ("dpmpp_sde", 3)
    assert np.array_equal(S._coef_table(S.ddim_timesteps, None), dpmpp_table(AC, G.karras_grid(AC.numpy(), 20), 3, 0.7))


def test_entry_point_rejects_bad_arguments_without_gpu():
    """vdb_dpmpp_sde_cfg_step refuses what vdb_dpmpp_cfg_step refuses, plus a missing seed and noise, a misaligned seed or noise
    and noise overlapping an output, before any launch (the fake addresses are never dereferenced)."""
    from vdb200._lib import lib
    n = 1024
    ok = dict(eu=0x100000, ec=0x200000, x=0x300000, coef=0x400000, idx=0x500000, hist=0x600000, xn=0x700000, dup=0x800000,
              p0=0x900000, n=n, seed=0xa00000, noise=0xb00000)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.vdb_dpmpp_sde_cfg_step(a["eu"], a["ec"], a["x"], a["coef"], a["idx"], 7.5, a["hist"], a["xn"], a["dup"],
                                          a["p0"], a["n"], a["seed"], a["noise"], None)

    before = lib.vdb_launch_count()
    for k in ("ec", "x", "coef", "idx", "hist", "xn"):
        assert call(**{k: None}) == 1, k
        assert b"dpmpp_sde_cfg_step: null" in lib.vdb_last_error()
    for n_bad in (0, -4):
        assert call(n=n_bad) == 1 and b"empty" in lib.vdb_last_error()
    assert call(seed=None, noise=None) == 1 and b"seed and noise" in lib.vdb_last_error()
    for k in ("eu", "ec", "x", "hist", "xn", "dup", "p0", "noise"):
        assert call(**{k: ok[k] + 4}) == 1, k
        assert b"16-byte aligned" in lib.vdb_last_error()
    for off in (1, 4):
        assert call(seed=ok["seed"] + off) == 1 and b"8-byte aligned" in lib.vdb_last_error()
    h = ok["hist"]
    for k in ("x", "xn", "dup", "p0"):
        for addr in (h, h + 4 * n, h + 4 * (3 * n - 4), h - 4 * (n - 4)):
            assert call(**{k: addr}) == 1, (k, addr)
            assert b"overlaps" in lib.vdb_last_error()
    # noise [noise, noise + n floats) against the ring and the outputs: first and last shared element
    for k, size in (("hist", 3 * n), ("xn", n), ("dup", n), ("p0", n)):
        for addr in (ok[k], ok[k] + 4 * (size - 4), ok[k] - 4 * (n - 4)):
            assert call(noise=addr) == 1, (k, addr)
            assert b"noise overlaps" in lib.vdb_last_error()
    assert lib.vdb_launch_count() == before


# ---- weak convergence of the oracle's SDE walk on the analytic Gaussian model --------------------------------------------------
MU, S_ = 0.3, 1.0


def _sde_moments(steps, order, eta, grid="uniform", n=100_000, seed=0):
    """Mean and variance of the oracle walk's output over n independent paths, x_T from the exact marginal at t_top."""
    ts = _ts(grid, steps)
    alpha, sigma = D.coefficients(AC.numpy(), ts)[:2]
    rng = np.random.default_rng(seed)
    x = MU * alpha[-1] + np.sqrt(alpha[-1] ** 2 * S_ * S_ + sigma[-1] ** 2) * rng.standard_normal(n)
    out = G.walk(x, lambda xv, i: D.gaussian_eps(xv, alpha[i], sigma[i], MU, S_), AC.numpy(), ts, order, eta=eta,
                 noise=lambda i: rng.standard_normal(n))
    return out.mean(), out.var()


def test_weak_convergence_on_the_analytic_model():
    """The exact marginal at ac[0] is N(alpha0 mu, alpha0^2 s^2 + sigma0^2).  The SDE walk's mean stays within its sampling error
    of it (one sigma of 1e5 draws: 3.2e-3), and the error of its variance falls with the step count: about as h for order 1 and
    faster for orders 2 and 3, whose long last steps on the uniform grid (eta = 1 doubles h in the phi functions) need 50 steps
    before they settle; the Karras grid at eta = 0.5 is within 0.01 at 50 steps."""
    a0 = float(AC[0])
    m_exact, v_exact = np.sqrt(a0) * MU, a0 * S_ * S_ + (1 - a0)
    for order in (1, 2, 3):
        errs = {}
        for steps in (50, 100, 200):
            m, v = _sde_moments(steps, order, 1.0)
            errs[steps] = v - v_exact
            assert abs(m - m_exact) <= 0.016, (order, steps, m - m_exact)
        print(f"order {order}, eta 1, uniform: variance error at 50 / 100 / 200 steps", {k: round(e, 4) for k, e in errs.items()})
        assert abs(errs[200]) < abs(errs[100]) < abs(errs[50]), order
        assert abs(errs[200]) <= (0.045 if order == 1 else 0.02), order
        m, v = _sde_moments(50, order, 0.5, grid="karras")
        print(f"order {order}, eta 0.5, karras, 50 steps: mean error {m - m_exact:.4f}, variance error {v - v_exact:.4f}")
        assert abs(m - m_exact) <= 0.016 and abs(v - v_exact) <= (0.12 if order == 1 else 0.01), order
