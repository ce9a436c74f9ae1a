"""Stochastic DPM-Solver++ on the GPU: vdb_dpmpp_sde_cfg_step bitwise against its fp32 op-order restatement with explicit noise and
against vdb_dpmpp_cfg_step where N = 0, its Philox draws, a device-counter walk on the analytic Gaussian model, DPMSolverSDESampler
(and the trailing / Karras grids of every fast sampler) on the mini UNet against the oracle fed the device draws, graph against
eager, seeds, and every sampling mode at eta = 0 (DPMSolverSampler bit for bit) and eta = 1."""
import numpy as np
import pytest
import torch

from oracle import dpm_sde_oracle as G
from oracle import dpm_solver_oracle as D
from oracle import vd_oracle as O
from test_dpm_solver_gpu import _data, _dev, restate
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
AC = O.ddpm_schedule(1000)["alphas_cumprod"]
F32 = np.float32


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _table(steps, order, eta, grid="uniform"):
    from lib.model_zoo.dpm_solver import dpmpp_table
    ts = G.grid(grid, steps, AC.numpy())
    return dpmpp_table(AC, ts, order, eta), ts


def draws(seed, i, n):
    """the kernel's Philox draws of grid index i for n elements, read back through a row whose only non-zero coefficient is N = 1
    (x' = ((0 x + 0 x0) + 1 z) = z exactly)"""
    from vdb200 import ops
    row = torch.zeros(i + 1, 8, device=DEV)
    row[i, 6] = 1.0
    z = torch.zeros(n, device=DEV)
    out = torch.empty(n, device=DEV)
    ops.dpmpp_cfg_step(None, z, z, row, _idx(i), 1.0, torch.empty(3 * n, device=DEV), x_next=out, seed=seed)
    return out


@pytest.mark.parametrize("order", [1, 2, 3])
def test_kernel_bitwise_with_explicit_noise_at_every_row(order):
    from vdb200 import ops
    t64, ts = _table(50, order, 1.0)
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    t32 = coef.cpu().numpy()
    g = np.random.default_rng(10 + order)
    for idx in range(50):
        v = idx % 8
        cfg, inplace, with_dup, with_p0 = v & 1, v & 2, v & 4, (v + 1) & 2
        n = (4099, 4096, 333, 1)[idx % 4]
        scale = 7.5 if cfg else 1.0
        eu, ec, x, hist = _data(g, n, idx, ts, cfg, scale)
        z = g.standard_normal(n).astype(F32)
        d_x, d_hist = _dev(x), _dev(hist.reshape(-1))
        x_next = d_x if inplace else torch.full((n,), float("nan"), device=DEV)
        dup = torch.full((n,), float("nan"), device=DEV) if with_dup else None
        p0 = torch.full((n,), float("nan"), device=DEV) if with_p0 else None
        ops.dpmpp_cfg_step(_dev(eu), _dev(ec), d_x, coef, _idx(idx), scale, d_hist, x_next=x_next, x_next_dup=dup, pred_x0=p0,
                           noise=_dev(z))
        want, want_x0 = restate(eu, ec, x, t32[idx], scale, hist[(idx + 1) % 3], hist[(idx + 2) % 3])
        N = F32(t32[idx, 6])
        if N != 0:
            want = want + N * z
        got = x_next.cpu().numpy()
        assert np.array_equal(got, want), (order, idx, np.abs(got - want).max())
        if with_dup:
            assert np.array_equal(dup.cpu().numpy(), want)
        if with_p0:
            assert np.array_equal(p0.cpu().numpy(), want_x0)
        ring = d_hist.view(3, n).cpu().numpy()
        assert np.array_equal(ring[idx % 3], want_x0)
        for s in ((idx + 1) % 3, (idx + 2) % 3):
            assert np.array_equal(ring[s], hist[s])


@pytest.mark.parametrize("order", [1, 2, 3])
def test_rows_without_noise_equal_the_deterministic_kernel(order):
    """eta = 0 rows, and the last row of an eta = 1 table, give vdb_dpmpp_cfg_step's bits with a seed or with noise given."""
    from vdb200 import ops
    g = np.random.default_rng(20 + order)
    t0, ts = _table(20, order, 0.0)
    t1, _ = _table(20, order, 1.0)
    for table, rows in ((t0, range(20)), (t1, [0])):
        coef = torch.tensor(table, dtype=torch.float32, device=DEV)
        for idx in rows:
            n = (4099, 4096, 333)[idx % 3]
            eu, ec, x, hist = _data(g, n, idx, ts, True, 7.5)
            outs = []
            for kw in ({}, {"seed": _seed(12345)}, {"noise": _dev(np.full(n, np.nan, F32))}):
                h = _dev(hist.reshape(-1))
                xn, p0 = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
                ops.dpmpp_cfg_step(_dev(eu), _dev(ec), _dev(x), coef, _idx(idx), 7.5, h, x_next=xn, pred_x0=p0, **kw)
                outs.append((xn.cpu(), p0.cpu(), h.cpu()))
            for o in outs[1:]:
                assert all(torch.equal(a, b) for a, b in zip(outs[0], o)), (order, idx)


def test_philox_draws():
    n = 1 << 20
    a = draws(_seed(7), 3, n)
    assert torch.equal(a, draws(_seed(7), 3, n)), "reproducible per (seed, step)"
    for other in (draws(_seed(7), 4, n), draws(_seed(8), 3, n)):
        assert (a != other).float().mean().item() > 0.999, "different across steps and seeds"
    q = a.view(-1, 4)
    assert (q[1:] != q[:-1]).all(dim=1).float().mean().item() > 0.999, "different across element quads"
    # tail elements of a length that is not a multiple of 4 are the draws of their quad
    assert torch.equal(draws(_seed(7), 3, 4099)[:4096], a[:4096])
    from vdb200 import ops
    ins = ops.inpaint_noise(_seed(7), _idx(3), 4096)
    assert (ins != a[:4096]).float().mean().item() > 0.999, "the SDE stream is not the inpainting stream"
    x = a.double()
    mean, var = x.mean().item(), x.var().item()
    print(f"[sde] {n} draws: mean {mean:.5f}, variance {var:.5f} (sampling sigma {1 / np.sqrt(n):.5f}, {np.sqrt(2 / n):.5f})")
    assert abs(mean) <= 5 / np.sqrt(n) and abs(var - 1) <= 5 * np.sqrt(2 / n)
    assert torch.isfinite(a).all()


@pytest.mark.parametrize("order", [1, 2, 3])
def test_device_walk_on_the_analytic_model(order):
    """The sampler's device loop without the UNet (the analytic eps by torch between launches, the step counter on the device,
    the Philox key in a device word) against the fp64 oracle walk fed the same draws."""
    from vdb200 import ops
    mu, s = 0.3, 1.0
    t64, ts = _table(30, order, 1.0, grid="karras")
    alpha, sigma = D.coefficients(AC, ts)[:2]
    n = 4096
    z0 = np.random.default_rng(1).standard_normal(n)
    x_start = mu * alpha[-1] + np.sqrt(alpha[-1] ** 2 * s * s + sigma[-1] ** 2) * z0
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    x = torch.tensor(x_start, dtype=torch.float32, device=DEV)
    hist = torch.empty(3 * n, device=DEV)
    idx = _idx(len(ts) - 1)
    seed = _seed(2024)
    xs = []
    for i in range(len(ts) - 1, -1, -1):
        a, gg = float(alpha[i]), float(sigma[i])
        eps = gg * (x - a * mu) / (a * a * s * s + gg * gg)
        ops.dpmpp_cfg_step(None, eps, x, coef, idx, 1.0, hist, x_next=x, seed=seed)
        ops.add_int(idx, -1)
        xs.append(x.double().cpu().numpy())
    trace = []
    G.walk(x_start, lambda xv, i: D.gaussian_eps(xv, alpha[i], sigma[i], mu, s), AC.numpy(), ts, order, eta=1.0,
           noise=lambda i: draws(seed, i, n).double().cpu().numpy(), trace=trace)
    for k, (got, (_, _, ref, _)) in enumerate(zip(xs, trace)):
        assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max(), (order, k, np.abs(got - ref).max())


# ---- the sampler on the mini UNet --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=7.5, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _noise_fn(S, shape):
    """the sampler's draws at grid index i, read back with the key it used, NHWC -> the oracle's layout"""
    key = S._st["sde_key"].clone()
    n = int(np.prod(shape))
    if len(shape) == 2:
        return lambda i: draws(key, i, n).view(*shape).double().cpu().numpy()
    bs, C, H, W = shape
    return lambda i: draws(key, i, n).view(bs, H, W, C).permute(0, 3, 1, 2).double().cpu().numpy()


@pytest.mark.parametrize("order,grid", [(2, "uniform"), (3, "uniform"), (2, "karras"), (3, "trailing")])
def test_sampler_vs_oracle(mini, order, grid):
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    net, sd, gi = mini
    S = DPMSolverSDESampler(net, order=order, grid=grid)
    with torch.no_grad():
        x, inter = S.sample(steps=8, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": gi["xT"]},
                            c_info=_cinfo(gi["c"], gi["u"]), verbose=False, log_every_t=1)
    assert len(inter["pred_x0"]) == len(G.grid(grid, 8, AC.numpy()))
    ref = G.sample(sd, gi["xT"], [gi["c"]], [gi["u"]], 8, order, 7.5, model_channels=64, grid_name=grid, eta=1.0,
                   noise=_noise_fn(S, [1, 4, 16, 16]))
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"8-step DPM-Solver++ {order}M SDE ({grid}) latent vs oracle")


def test_sampler_multicontext_vs_oracle(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(5)
    ct, ut = torch.randn(1, 77, 768, generator=g) * 0.5, torch.randn(1, 77, 768, generator=g) * 0.5
    ci, ui = torch.randn(1, 257, 768, generator=g) * 0.5, torch.zeros(1, 257, 768)
    S = DPMSolverSDESampler(net, order=3, grid="karras")
    with torch.no_grad():
        x, _ = S.sample_multicontext(steps=6, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": gi["xT"]},
                                     c_info_list=[_cinfo(ct, ut, ratio=0.7), _cinfo(ci, ui, typ="image", ratio=0.3)],
                                     verbose=False, eta=0.5)
    ref = G.sample(sd, gi["xT"], [ct, ci], [ut, ui], 6, 3, 7.5, c_types=("text", "image"), ratios=[0.7, 0.3], model_channels=64,
                   grid_name="karras", eta=0.5, noise=_noise_fn(S, [1, 4, 16, 16]))
    _cmp(x, ref, cos_min=0.995, tol=0.1, what="6-step dual-context 3M SDE (karras, eta 0.5) latent vs oracle")


def test_sampler_text_latent_vs_oracle():
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    net, sd = build_net(mini=True, with_vae=False, text_flows=True)
    g = torch.Generator().manual_seed(41)
    xT = torch.randn(2, 768, generator=g)
    c, u = torch.randn(2, 257, 768, generator=g) * 0.5, torch.zeros(2, 257, 768)
    outs = []
    for graph in (False, True):
        S = DPMSolverSDESampler(net, use_cuda_graph=graph)
        torch.manual_seed(3)
        with torch.no_grad():
            x, _ = S.sample(steps=6, shape=[2, 768], x_info={"type": "text", "xt": xT.clone()}, c_info=_cinfo(c, u, typ="image"),
                            verbose=False)
        assert x.shape == (2, 768)
        outs.append(x)
    assert torch.equal(outs[0], outs[1]), "graph path must equal the eager path"
    ref = G.sample(sd, xT, [c], [u], 6, 2, 7.5, c_types=("image",), text=True, model_channels=64, eta=1.0,
                   noise=_noise_fn(S, [2, 768]))
    _cmp(outs[0], ref, cos_min=0.995, tol=0.1, what="6-step 2M SDE on a text latent (i2t) vs oracle")


def test_sampler_img2img_start_vs_oracle(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(11)
    x0 = torch.randn(1, 4, 16, 16, generator=g) * 0.8
    noise = torch.randn(1, 4, 16, 16, generator=g)
    steps, k = 10, 6
    orig = net.q_sample
    net.q_sample = lambda x_start, t, noise_=None: orig(x_start, t, noise=noise.to(x_start.device))   # inject the draw
    S = DPMSolverSDESampler(net, order=2, grid="trailing")
    try:
        with torch.no_grad():
            x, inter = S.sample(steps=steps, shape=[1, 4, 16, 16], c_info=_cinfo(gi["c"], gi["u"]), verbose=False, log_every_t=1,
                                x_info={"type": "image", "x0": x0.to(DEV), "x0_forward_timesteps": k})
    finally:
        net.q_sample = orig
    assert len(inter["pred_x0"]) == k
    ref = G.sample(sd, None, [gi["c"]], [gi["u"]], steps, 2, 7.5, model_channels=64, x0=x0, x0_forward_timesteps=k, x0_noise=noise,
                   grid_name="trailing", eta=1.0, noise=_noise_fn(S, [1, 4, 16, 16]))
    _cmp(x, ref, cos_min=0.995, tol=0.1, what="img2img 6-of-10-step 2M SDE (trailing) latent vs oracle")


@pytest.mark.parametrize("grid", ["trailing", "karras"])
@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_deterministic_samplers_on_the_new_grids(mini, kind, grid):
    """DDIM (order 1 of the oracle: DDIM at eta 0) and DPM-Solver++ 2M walk the grid they are given."""
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    S = DDIMSampler(net, grid=grid) if kind == "ddim" else DPMSolverSampler(net, order=2, grid=grid)
    with torch.no_grad():
        x, _ = S.sample(steps=8, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": gi["xT"]}, c_info=_cinfo(gi["c"], gi["u"]),
                        verbose=False, eta=0.)
    ref = G.sample(sd, gi["xT"], [gi["c"]], [gi["u"]], 8, 1 if kind == "ddim" else 2, 7.5, model_channels=64, grid_name=grid)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"8-step {kind} on the {grid} grid vs oracle")


def test_graph_equals_eager_and_seeds(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(3)
    xT = torch.randn(2, 4, 16, 16, generator=g)
    c, u = torch.randn(2, 77, 768, generator=g).to(DEV), torch.randn(2, 77, 768, generator=g).to(DEV)

    def run(S, seed, eta=1.0):
        torch.manual_seed(seed)
        with torch.no_grad():
            return S.sample(steps=6, shape=[2, 4, 16, 16], x_info={"type": "image", "xt": xT.clone()}, verbose=False, eta=eta,
                            c_info={"type": "text", "conditioning": c, "unconditional_conditioning": u,
                                    "unconditional_guidance_scale": 5.0})[0]
    for order in (2, 3):
        eager = run(DPMSolverSDESampler(net, order=order, use_cuda_graph=False, grid="karras"), 0)
        Sg = DPMSolverSDESampler(net, order=order, grid="karras")
        g1 = run(Sg, 0)
        assert torch.equal(eager, g1), "graph path must be bit-identical to the eager path"
        assert torch.equal(run(Sg, 0), g1), "the same seed gives the same latent"
        g2 = run(Sg, 1)
        assert not torch.equal(g1, g2) and (g1 - g2).abs().max().item() > 1e-3, "another seed gives another latent"
        assert torch.equal(g2, run(DPMSolverSDESampler(net, order=order, use_cuda_graph=False, grid="karras"), 1))
        # eta changes only the table: the cached graph replays and still equals the eager path
        n_graphs = len(Sg._graphs)
        g3 = run(Sg, 2, eta=0.4)
        assert torch.equal(g3, run(DPMSolverSDESampler(net, order=order, use_cuda_graph=False, grid="karras"), 2, eta=0.4))
        assert len(Sg._graphs) == n_graphs and torch.isfinite(g3).all()


# ---- modes ---------------------------------------------------------------------------------------------------------------------
def _mode_inputs(kind, net, gi):
    """-> (x_info builder, c_info list, shape, steps) of one sampling mode on the mini UNet"""
    from lib.model_zoo.ddim import DDIMSampler
    g = torch.Generator().manual_seed(29)
    bs, C, H, W = 2, 4, 16, 16
    steps = 6
    c = (gi["c"] + 0.2 * torch.randn(bs, 77, 768, generator=g)).to(DEV)
    u = gi["u"].repeat(bs, 1, 1).to(DEV)
    cl = [_cinfo(c, u)]
    xT = torch.randn(bs, C, H, W, generator=g).to(DEV)
    x0 = (torch.randn(bs, C, H, W, generator=g) * 0.8).to(DEV)
    mask = torch.zeros(bs, 1, H, W)
    mask[..., W // 2:] = 1.0
    mask = mask.to(DEV)
    if kind == "plain":
        return lambda: {"type": "image", "xt": xT.clone()}, cl, [bs, C, H, W], steps
    if kind == "inpaint":
        return lambda: {"type": "image", "xt": xT.clone(), "x0": x0, "inpaint_mask": mask}, cl, [bs, C, H, W], steps
    if kind == "inversion":
        with torch.no_grad():
            inv = DDIMSampler(net).invert(steps, x0, _cinfo(c, u, scale=1.0), k=4)
        return lambda: {"type": "image", "inversion": inv, "inpaint_mask": mask}, cl, [bs, C, H, W], steps
    if kind == "regions":
        from lib.model_zoo.regions import Region, Regions
        rm = torch.zeros(1, H, W, device=DEV)
        rm[:, :H // 2] = 1.0
        reg = Regions([Region(rm, (gi["c"] * 0.5).repeat(bs, 1, 1).to(DEV))])
        return lambda: {"type": "image", "xt": xT.clone(), "regions": reg}, cl, [bs, C, H, W], steps
    if kind == "sag":
        from lib.model_zoo.sag import SelfAttentionGuidance
        return lambda: {"type": "image", "xt": xT.clone(), "sag": SelfAttentionGuidance(0.75)}, cl, [bs, C, H, W], steps
    from test_prompt_edit_gpu import _contexts, _edit
    ed, _, _ = _edit("replace", True)
    _, _, _, cl_fn = _contexts(3, False, g)
    xt3 = torch.randn(1, C, H, W, generator=g).expand(3, C, H, W).contiguous().to(DEV)
    return lambda: {"type": "image", "xt": xt3}, cl_fn(ed), [3, C, H, W], steps


def _run(S, x_info, cl, shape, steps, eta=None, seed=0):
    kw = dict(steps=steps, shape=shape, x_info=x_info, verbose=False)
    if eta is not None:
        kw["eta"] = eta
    torch.manual_seed(seed)
    with torch.no_grad():
        return (S.sample_multicontext(c_info_list=cl, **kw) if len(cl) > 1 else S.sample(c_info=cl[0], **kw))[0]


@pytest.mark.parametrize("kind", ["plain", "inpaint", "inversion", "regions", "sag", "prompt_edit"])
def test_modes(mini, kind):
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler
    net, sd, gi = mini
    xi, cl, shape, steps = _mode_inputs(kind, net, gi)
    # eta = 0: DPMSolverSampler bit for bit, with the same launches per step
    Sp, S0 = DPMSolverSampler(net, order=2), DPMSolverSDESampler(net, order=2)
    ref = _run(Sp, xi(), cl, shape, steps, eta=0.)
    got = _run(S0, xi(), cl, shape, steps, eta=0.)
    assert torch.equal(got, ref), kind
    assert S0.last_step_launches == Sp.last_step_launches > 0, (S0.last_step_launches, Sp.last_step_launches)
    print(f"[sde] {kind}: launches per step {S0.last_step_launches}")
    # eta = 1: graph equals eager, finite, and different from eta = 0
    S1 = DPMSolverSDESampler(net, order=2)
    g1 = _run(S1, xi(), cl, shape, steps, seed=5)
    e1 = _run(DPMSolverSDESampler(net, order=2, use_cuda_graph=False), xi(), cl, shape, steps, seed=5)
    assert torch.equal(g1, e1), kind
    assert torch.isfinite(g1).all() and not torch.equal(g1, ref), kind
    assert S1.last_step_launches == Sp.last_step_launches
    if kind in ("inpaint", "inversion"):
        # a hard mask returns x0 exactly where it keeps (the inversion's slot 0 is x0)
        x0 = xi()["x0"] if kind == "inpaint" else xi()["inversion"].trajectory[0]
        x0 = x0 if kind == "inpaint" else x0.permute(0, 3, 1, 2)
        W = shape[3]
        assert torch.equal(g1[..., :W // 2].float(), x0[..., :W // 2].float()), kind
