"""DPM-Solver++ sampler, CPU side: the folded per-step table (lib/model_zoo/dpm_solver.py) against the fp64 oracle that steps with
lambda, expm1 and a history list (oracle/dpm_solver_oracle.py); order 1 against the DDIM oracle update; convergence orders on the
analytic Gaussian model; the order-per-step rule; the argument checks of the sampler and of vdb_dpmpp_cfg_step."""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import dpm_solver_oracle as D
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]          # the model's fp32 buffer
MU, S = 0.3, 1.0


def _table(steps, order, walk=None):
    from lib.model_zoo.dpm_solver import dpmpp_table
    ts = O.make_ddim_timesteps(steps)[:walk]
    return dpmpp_table(AC, ts, order), ts


def table_walk(table, x, eps_fn):
    """The kernel's arithmetic in fp64: x0 = P x + Q e, x' = A x + B x0_i + C x0_{i+1} + D x0_{i+2}; -> x' of every step."""
    hist, out = {}, []
    for i in range(table.shape[0] - 1, -1, -1):
        P, Q, A, B, C, Dd = table[i, :6]
        x0 = P * x + Q * eps_fn(x, i)
        x = A * x + B * x0
        if C != 0:
            x = x + C * hist[i + 1]
        if Dd != 0:
            x = x + Dd * hist[i + 2]
        hist[i] = x0
        out.append(x)
    return out


def _eps_fn(ts, wobble=0.05):
    """the analytic Gaussian eps plus a non-linear term, so the walk is not affine in x_T"""
    alpha, sigma = D.coefficients(AC, ts)[:2]
    return lambda x, i: D.gaussian_eps(x, alpha[i], sigma[i], MU, S) + wobble * np.sin(3.0 * x)


def _z(n=1000):
    return np.random.default_rng(0).standard_normal(n)


def _start(ts, z):
    alpha, sigma = D.coefficients(AC, ts)[:2]
    return MU * alpha[-1] + np.sqrt(alpha[-1] ** 2 * S * S + sigma[-1] ** 2) * z


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("steps,walk", [(5, None), (13, None), (14, None), (15, None), (50, None), (50, 30), (20, 12)])
def test_table_matches_the_oracle_step_for_step(order, steps, walk):
    table, ts = _table(steps, order, walk)
    assert table.shape == (len(ts), 8) and not table[:, 6:].any()
    x = _start(ts, _z(257))
    trace = []
    D.walk(x, _eps_fn(ts), AC.numpy(), ts, order, trace=trace)
    mine = table_walk(table, x, _eps_fn(ts))
    assert len(mine) == len(trace) == len(ts)
    for k, ((_, _, ref), got) in enumerate(zip(trace, mine)):
        err = np.abs(got - ref).max() / np.abs(ref).max()
        assert err <= 1e-12, (k, err)


def test_order_one_is_the_ddim_oracle_update(monkeypatch):
    """Order 1 against vd_oracle.p_sample_ddim (its model call replaced by the given e), in fp64.  The oracle's schedule rounds
    sqrt(1 - a_t) to fp32 as the reference does; the fp64 comparison gives it the exact value."""
    steps = 50
    table, ts = _table(steps, 1)
    assert not table[:, 4:].any()
    sched = O.ddim_schedule(AC, steps)
    exact = dict(sched, sqrt_one_minus_alphas=np.sqrt(1.0 - sched["alphas"].astype(np.float64)))
    g = np.random.default_rng(1)
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        for i in range(steps):
            x, e = torch.from_numpy(g.standard_normal((2, 4, 3, 3))), torch.from_numpy(g.standard_normal((2, 4, 3, 3)))
            monkeypatch.setattr(O, "apply_model", lambda *a, **k: e)
            ref, ref_x0, _ = O.p_sample_ddim(None, x, [None], [None], None, i, exact, 1.0)
            P, Q, A, B = table[i, :4]
            x0 = P * x.numpy() + Q * e.numpy()
            got = A * x.numpy() + B * x0
            assert np.abs(x0 - ref_x0.numpy()).max() <= 1e-12 * np.abs(ref_x0.numpy()).max(), i
            assert np.abs(got - ref.numpy()).max() <= 1e-12 * np.abs(ref.numpy()).max(), i
    finally:
        torch.set_default_dtype(old)


def _ddim_err(steps, z):
    """fp64 DDIM (the oracle's update with exact square roots) on the analytic model: max error against the exact solution"""
    sched = O.ddim_schedule(AC, steps)
    a, ap = sched["alphas"].astype(np.float64), sched["alphas_prev"].astype(np.float64)
    ts = sched["timesteps"]
    x = _start(ts, z)
    for i in range(steps - 1, -1, -1):
        e = D.gaussian_eps(x, np.sqrt(a[i]), np.sqrt(1 - a[i]), MU, S)
        x0 = (x - np.sqrt(1 - a[i]) * e) / np.sqrt(a[i])
        x = np.sqrt(ap[i]) * x0 + np.sqrt(1 - ap[i]) * e
    return np.abs(x - _exact(ts, z)).max()


def _exact(ts, z):
    alpha, sigma, _, _, _ = D.coefficients(AC, ts)
    a0 = float(AC[0])
    return D.gaussian_exact(_start(ts, z), alpha[-1], sigma[-1], np.sqrt(a0), np.sqrt(1 - a0), MU, S)


def _solver_err(steps, order, z):
    table, ts = _table(steps, order)
    x = table_walk(table, _start(ts, z), _eps_fn(ts, wobble=0.0))[-1]
    return np.abs(x - _exact(ts, z)).max()


def test_convergence_order_on_the_analytic_model():
    z = _z()
    observed = {o: np.log2(_solver_err(250, o, z) / _solver_err(500, o, z)) for o in (1, 2, 3)}
    print("observed orders (250 / 500 steps):", {o: round(v, 3) for o, v in observed.items()})
    assert 0.9 <= observed[1] <= 1.1
    assert observed[2] >= 1.5
    assert observed[3] >= 2.5


def test_error_table_of_the_analytic_model():
    """Max error of the final sample against the exact probability-flow solution, data N(0.3, 1), x_T from 1000 seeded draws."""
    z = _z()
    want = {20: (0.246, 0.176, 0.127), 25: (0.200, 0.125, 0.088), 50: (0.103, 0.042, 0.023)}
    for steps, (ddim, m2, m3) in want.items():
        got = (_ddim_err(steps, z), _solver_err(steps, 2, z), _solver_err(steps, 3, z))
        print(steps, ["%.4f" % v for v in got])
        for g, w in zip(got, (ddim, m2, m3)):
            assert abs(g - w) <= 5.01e-4, (steps, got)
        assert abs(_solver_err(steps, 1, z) - got[0]) <= 1e-12        # first order is DDIM


def test_order_per_step():
    from lib.model_zoo.dpm_solver import step_order
    # warm-up: the first steps use the history they have
    assert [step_order(3, k, 49 - k, 50) for k in range(4)] == [1, 2, 3, 3]
    assert [step_order(2, k, 49 - k, 50) for k in range(3)] == [1, 2, 2]
    # 15 steps or more: no lower-order final steps; fewer: the last steps drop order
    assert [step_order(3, 14 - i, i, 15) for i in range(3)] == [3, 3, 3]
    assert [step_order(3, 13 - i, i, 14) for i in range(3)] == [1, 2, 3]
    assert [step_order(2, 13 - i, i, 14) for i in range(2)] == [1, 2]
    # the table carries the rule: C (x0_{i+1}) and D (x0_{i+2}) are exactly zero where the order does not reach them.  The walk
    # is DDIM's grid, range(0, 1000, 1000 // steps) + 1: 14 or 15 steps walk 15 or 16 points, 13 steps walk 14
    for steps, order, walk_len in ((50, 3, 50), (15, 3, 16), (14, 3, 15), (13, 3, 14), (5, 3, 5), (13, 2, 14), (14, 2, 15),
                                   (50, 1, 50)):
        table, _ = _table(steps, order)
        assert table.shape[0] == walk_len
        for i in range(walk_len):
            o = step_order(order, walk_len - 1 - i, i, walk_len)
            assert (table[i, 4] != 0) == (o >= 2) and (table[i, 5] != 0) == (o >= 3), (steps, order, i)
        assert (table[0, 4] != 0) == (walk_len >= 15 and order >= 2)
    # an img2img walk of 6 steps out of 50: the walk's length decides
    table, _ = _table(50, 3, 6)
    assert [(table[i, 4] != 0, table[i, 5] != 0) for i in range(6)] == [(False, False), (True, False)] + [(True, True)] * 2 + \
        [(True, False), (False, False)]


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def test_sampler_argument_checks():
    from lib.model_zoo.dpm_solver import DPMSolverSampler, dpmpp_table
    for bad in (0, 4, "2"):
        with pytest.raises(ValueError, match="order"):
            DPMSolverSampler(_fake_model(), order=bad)
        with pytest.raises(ValueError, match="order"):
            dpmpp_table(AC, O.make_ddim_timesteps(10), bad)
    S = DPMSolverSampler(_fake_model())
    assert S.order == 2
    c = {"type": "text", "conditioning": torch.zeros(1, 77, 768), "unconditional_conditioning": torch.zeros(1, 77, 768),
         "unconditional_guidance_scale": 7.5}
    with pytest.raises(ValueError, match="eta"):
        S.sample(steps=10, shape=[1, 4, 8, 8], x_info={"type": "image"}, c_info=c, eta=0.5, verbose=False)
    with pytest.raises(ValueError, match="eta"):
        S.sample_multicontext(steps=10, shape=[1, 4, 8, 8], x_info={"type": "image"}, c_info_list=[c], eta=1.0, verbose=False)
    with pytest.raises(NotImplementedError):
        S.p_sample_ddim({"x": None}, c, None, 0)
    with pytest.raises(NotImplementedError):
        S.p_sample_ddim_multicontext({"x": None}, [c], None, 0)
    S.make_schedule(10, verbose=False)
    assert S._coef_table(S.ddim_timesteps, None).shape == (10, 8) and S._graph_tag() == ("dpmpp", 2)


def test_entry_point_rejects_bad_arguments_without_gpu():
    """vdb_dpmpp_cfg_step refuses null, misaligned, empty and overlapping arguments before any launch (the fake addresses below
    are never dereferenced: every call here fails its checks)."""
    from vdb200._lib import lib
    n = 1024
    ok = dict(eu=0x100000, ec=0x200000, x=0x300000, coef=0x400000, idx=0x500000, hist=0x600000, xn=0x700000, dup=0x800000,
              p0=0x900000, n=n)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.vdb_dpmpp_cfg_step(a["eu"], a["ec"], a["x"], a["coef"], a["idx"], 7.5, a["hist"], a["xn"], a["dup"], a["p0"],
                                      a["n"], None)

    before = lib.vdb_launch_count()
    for k in ("ec", "x", "coef", "idx", "hist", "xn"):
        assert call(**{k: None}) == 1, k
        assert b"dpmpp_cfg_step: null" in lib.vdb_last_error()
    for n_bad in (0, -4):
        assert call(n=n_bad) == 1 and b"empty" in lib.vdb_last_error()
    for k in ("eu", "ec", "x", "hist", "xn", "dup", "p0"):
        assert call(**{k: ok[k] + 4}) == 1, k
        assert b"16-byte aligned" in lib.vdb_last_error()
    # the ring [hist, hist + 3n floats) against x, x_next, x_next_dup and pred_x0: first and last shared element, inside
    h = ok["hist"]
    for k in ("x", "xn", "dup", "p0"):
        for addr in (h, h + 4 * n, h + 4 * (3 * n - 4), h - 4 * (n - 4)):
            assert call(**{k: addr}) == 1, (k, addr)
            assert b"overlaps" in lib.vdb_last_error()
    assert lib.vdb_launch_count() == before
