"""DPM-Solver++ on the GPU: vdb_dpmpp_cfg_step bitwise against its fp32 op-order restatement and against fp64, order 1 against
K4 (vdb_ddim_cfg_step), a device-counter walk on the analytic Gaussian model, and DPMSolverSampler on the mini UNet against the
oracle (vd_oracle's UNet + the fp64 solver of oracle/dpm_solver_oracle.py), against DDIMSampler at order 1, graph against eager."""
import numpy as np
import pytest
import torch

from oracle import dpm_solver_oracle as D
from oracle import vd_oracle as O
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
AC = O.ddpm_schedule(1000)["alphas_cumprod"]
F32 = np.float32


def _table64(steps, order):
    from lib.model_zoo.dpm_solver import dpmpp_table
    ts = O.make_ddim_timesteps(steps)
    return dpmpp_table(AC, ts, order), ts


def restate(eu, ec, x, row, scale, h1, h2):
    """the header's op order in numpy fp32 (every op rounded to nearest) -> (x_next, x0)"""
    P, Q, A, B, C, Dd = (F32(v) for v in row[:6])
    e = ec if eu is None else eu + F32(scale) * (ec - eu)
    x0 = P * x + Q * e
    v = A * x + B * x0
    if C != 0:
        v = v + C * h1
    if Dd != 0:
        v = v + Dd * h2
    return v, x0


def _data(g, n, idx, ts, cfg, scale):
    """x = alpha x0 + sigma eps at grid index idx with x0, eps ~ N(0, 1); e_c - e_u small as in guided sampling; ring of x0s"""
    alpha, sigma = D.coefficients(AC, ts)[:2]
    x0, eps = g.standard_normal(n), g.standard_normal(n)
    x = (alpha[idx] * x0 + sigma[idx] * eps).astype(F32)
    if cfg:
        eu = (eps + 0.05 * g.standard_normal(n)).astype(F32)
        ec = (eu + (eps - eu) / scale).astype(F32)
    else:
        eu, ec = None, eps.astype(F32)
    hist = (x0[None] + 0.1 * g.standard_normal((3, n))).astype(F32)
    return eu, ec, x, hist


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("order", [1, 2, 3])
def test_kernel_bitwise_and_against_fp64_at_every_row(order):
    from vdb200 import ops
    t64, ts = _table64(50, order)
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    t32 = coef.cpu().numpy()
    g = np.random.default_rng(order)
    worst = 0.0
    for idx in range(50):
        v = idx % 8
        cfg, inplace, with_dup, with_p0 = v & 1, v & 2, v & 4, (v + 1) & 2
        n = (4099, 4096, 333, 1)[idx % 4]
        scale = 7.5 if cfg else 1.0
        eu, ec, x, hist = _data(g, n, idx, ts, cfg, scale)
        d_eu, d_ec, d_x, d_hist = _dev(eu), _dev(ec), _dev(x), _dev(hist.reshape(-1))
        x_next = d_x if inplace else torch.full((n,), float("nan"), device=DEV)
        dup = torch.full((n,), float("nan"), device=DEV) if with_dup else None
        p0 = torch.full((n,), float("nan"), device=DEV) if with_p0 else None
        sidx = torch.tensor([idx], dtype=torch.int32, device=DEV)
        ops.dpmpp_cfg_step(d_eu, d_ec, d_x, coef, sidx, scale, d_hist, x_next=x_next, x_next_dup=dup, pred_x0=p0)
        want, want_x0 = restate(eu, ec, x, t32[idx], scale, hist[(idx + 1) % 3], hist[(idx + 2) % 3])
        got = x_next.cpu().numpy()
        assert np.array_equal(got, want), (order, idx, np.abs(got - want).max())
        if with_dup:
            assert np.array_equal(dup.cpu().numpy(), want)
        if with_p0:
            assert np.array_equal(p0.cpu().numpy(), want_x0)
        ring = d_hist.view(3, n).cpu().numpy()
        assert np.array_equal(ring[idx % 3], want_x0)
        for s in ((idx + 1) % 3, (idx + 2) % 3):
            assert np.array_equal(ring[s], hist[s]), "only slot idx % 3 is written"
        # fp64: the same step with the fp64 table on the same fp32 inputs
        P, Q, A, B, C, Dd = t64[idx, :6]
        e64 = ec.astype(np.float64) if eu is None else eu + scale * (ec.astype(np.float64) - eu)
        x064 = P * x + Q * e64
        ref = A * x + B * x064 + C * hist[(idx + 1) % 3] + Dd * hist[(idx + 2) % 3]
        rel = np.abs(got - ref).max() / np.abs(ref).max()
        worst = max(worst, rel)
        assert rel <= 1e-5, (order, idx, rel)
    print(f"[dpm] order {order}: kernel vs fp64 worst {worst:.3g} of max|x'|")


@pytest.mark.parametrize("order", [2, 3])
def test_nan_ring_is_not_read_at_the_first_steps(order):
    """A ring full of NaN at the first step (and the slot not yet written at the second step of 3M) leaves the output finite."""
    from vdb200 import ops
    t64, ts = _table64(50, order)
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    g = np.random.default_rng(7)
    n = 1027
    hist = torch.full((3 * n,), float("nan"), device=DEV)
    for k, idx in enumerate((49, 48)):
        eu, ec, x, _ = _data(g, n, idx, ts, True, 7.5)
        out, p0 = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        ops.dpmpp_cfg_step(_dev(eu), _dev(ec), _dev(x), coef, torch.tensor([idx], dtype=torch.int32, device=DEV), 7.5, hist,
                           x_next=out, pred_x0=p0)
        assert torch.isfinite(out).all() and torch.isfinite(p0).all(), (order, idx)
        if order == 2:
            break


def test_order_one_against_k4_at_every_step():
    """With the order-1 table the kernel is DDIM: against vdb_ddim_cfg_step on the same inputs, within 2^-20 of max|x_prev|."""
    from vdb200 import ops
    t64, ts = _table64(50, 1)
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    sch = O.ddim_schedule(AC, 50)
    k4 = torch.tensor(np.stack([sch["alphas"], sch["alphas_prev"], sch["sigmas"], sch["sqrt_one_minus_alphas"]], 1),
                      dtype=torch.float32, device=DEV).contiguous()
    g = np.random.default_rng(3)
    n = 4096
    worst = 0.0
    hist = torch.zeros(3 * n, device=DEV)
    for idx in range(50):
        eu, ec, x, _ = _data(g, n, idx, ts, True, 7.5)
        sidx = torch.tensor([idx], dtype=torch.int32, device=DEV)
        a, _ = ops.dpmpp_cfg_step(_dev(eu), _dev(ec), _dev(x), coef, sidx, 7.5, hist)
        b, _ = ops.ddim_cfg_step(_dev(eu), _dev(ec), _dev(x), k4, 7.5, step_idx=sidx)
        rel = (a - b).abs().max().item() / b.abs().max().item()
        worst = max(worst, rel)
        assert rel <= 2.0 ** -20, (idx, rel)
    print(f"[dpm] order 1 vs K4: worst {worst:.3g} of max|x_prev| (2^-20 = {2.0 ** -20:.3g})")


def _device_walk(steps, order, z, mu=0.3, s=1.0, trace=None):
    """the sampler's device loop without the UNet: the analytic eps by torch between launches, the step counter on the device"""
    from vdb200 import ops
    t64, ts = _table64(steps, order)
    alpha, sigma = D.coefficients(AC, ts)[:2]
    n = z.shape[0]
    coef = torch.tensor(t64, dtype=torch.float32, device=DEV)
    x = torch.tensor(mu * alpha[-1] + np.sqrt(alpha[-1] ** 2 * s * s + sigma[-1] ** 2) * z, dtype=torch.float32, device=DEV)
    hist = torch.empty(3 * n, device=DEV)
    idx = torch.tensor([len(ts) - 1], dtype=torch.int32, device=DEV)
    xs = []
    for i in range(len(ts) - 1, -1, -1):
        a, g = float(alpha[i]), float(sigma[i])
        eps = g * (x - a * mu) / (a * a * s * s + g * g)
        ops.dpmpp_cfg_step(None, eps, x, coef, idx, 1.0, hist, x_next=x)
        ops.add_int(idx, -1)
        if trace is not None:
            xs.append(x.double().cpu().numpy())
    assert int(idx.item()) == -1
    return x.double().cpu().numpy(), xs, ts


@pytest.mark.parametrize("order", [1, 2, 3])
def test_device_walk_on_the_analytic_model(order):
    z = np.random.default_rng(0).standard_normal(1000)
    mu, s = 0.3, 1.0
    x, xs, ts = _device_walk(50, order, z, trace=True)
    alpha, sigma = D.coefficients(AC, ts)[:2]
    trace = []
    D.walk(mu * alpha[-1] + np.sqrt(alpha[-1] ** 2 * s * s + sigma[-1] ** 2) * z,
           lambda xv, i: D.gaussian_eps(xv, alpha[i], sigma[i], mu, s), AC.numpy(), ts, order, trace=trace)
    for k, (got, (_, _, ref)) in enumerate(zip(xs, trace)):
        assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max(), (order, k)
    # convergence order of the device walk against the exact probability-flow solution
    a0 = float(AC[0])

    def err(steps):
        xe, _, tse = _device_walk(steps, order, z)
        al, sg = D.coefficients(AC, tse)[:2]
        x_t = mu * al[-1] + np.sqrt(al[-1] ** 2 * s * s + sg[-1] ** 2) * z
        return np.abs(xe - D.gaussian_exact(x_t, al[-1], sg[-1], np.sqrt(a0), np.sqrt(1 - a0), mu, s)).max()
    observed = np.log2(err(250) / err(500))
    print(f"[dpm] device walk, order {order}: observed order {observed:.3f} (250 / 500 steps)")
    lo, hi = {1: (0.9, 1.1), 2: (1.5, 9), 3: (2.5, 9)}[order]
    assert lo <= observed <= hi


# ---- the sampler on the mini UNet --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=7.5, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


@pytest.mark.parametrize("order", [1, 2, 3])
def test_sampler_vs_oracle(mini, order):
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    with torch.no_grad():
        x, inter = DPMSolverSampler(net, order=order).sample(steps=6, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": gi["xT"]},
                                                             c_info=_cinfo(gi["c"], gi["u"]), verbose=False, eta=0., log_every_t=1)
    ref = D.sample(sd, gi["xT"], [gi["c"]], [gi["u"]], 6, order, 7.5, model_channels=64)
    # DDIM's grid for 6 steps, range(0, 1000, 166) + 1, has 7 points: the walk logs every one of them
    assert len(inter["pred_x0"]) == len(inter["pred_xt"]) == len(O.make_ddim_timesteps(6)) == 7
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"6-step DPM-Solver++ order {order} final latent vs oracle")


def test_sampler_multicontext_vs_oracle(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(5)
    ct, ut = torch.randn(1, 77, 768, generator=g) * 0.5, torch.randn(1, 77, 768, generator=g) * 0.5
    ci, ui = torch.randn(1, 257, 768, generator=g) * 0.5, torch.zeros(1, 257, 768)
    with torch.no_grad():
        x, _ = DPMSolverSampler(net, order=3).sample_multicontext(
            steps=5, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": gi["xT"]},
            c_info_list=[_cinfo(ct, ut, ratio=0.7), _cinfo(ci, ui, typ="image", ratio=0.3)], verbose=False, eta=0.)
    ref = D.sample(sd, gi["xT"], [ct, ci], [ut, ui], 5, 3, 7.5, c_types=("text", "image"), ratios=[0.7, 0.3], model_channels=64)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what="5-step dual-context DPM-Solver++ 3M latent vs oracle")


def test_sampler_text_latent_vs_oracle():
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd = build_net(mini=True, with_vae=False, text_flows=True)
    g = torch.Generator().manual_seed(41)
    xT = torch.randn(2, 768, generator=g)
    c, u = torch.randn(2, 257, 768, generator=g) * 0.5, torch.zeros(2, 257, 768)
    outs = []
    for graph in (False, True):
        with torch.no_grad():
            x, _ = DPMSolverSampler(net, use_cuda_graph=graph).sample(
                steps=5, shape=[2, 768], x_info={"type": "text", "xt": xT.clone()}, c_info=_cinfo(c, u, typ="image"),
                verbose=False, eta=0.)
        assert x.shape == (2, 768)
        outs.append(x)
    assert torch.equal(outs[0], outs[1]), "graph path must equal the eager path"
    ref = D.sample(sd, xT, [c], [u], 5, 2, 7.5, c_types=("image",), text=True, model_channels=64)
    _cmp(outs[0], ref, cos_min=0.995, tol=0.1, what="5-step DPM-Solver++ 2M on a text latent (i2t) vs oracle")


def test_sampler_img2img_start_vs_oracle(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(11)
    x0 = torch.randn(1, 4, 16, 16, generator=g) * 0.8
    noise = torch.randn(1, 4, 16, 16, generator=g)
    steps, k = 8, 5
    orig = net.q_sample
    net.q_sample = lambda x_start, t, noise_=None: orig(x_start, t, noise=noise.to(x_start.device))   # inject the draw
    try:
        with torch.no_grad():
            x, inter = DPMSolverSampler(net, order=3).sample(
                steps=steps, shape=[1, 4, 16, 16], x_info={"type": "image", "x0": x0.to(DEV), "x0_forward_timesteps": k},
                c_info=_cinfo(gi["c"], gi["u"]), verbose=False, eta=0., log_every_t=1)
    finally:
        net.q_sample = orig
    assert len(inter["pred_x0"]) == k, "the img2img walk covers exactly x0_forward_timesteps steps"
    ref = D.sample(sd, None, [gi["c"]], [gi["u"]], steps, 3, 7.5, model_channels=64, x0=x0, x0_forward_timesteps=k, x0_noise=noise)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what="img2img 5-of-8-step DPM-Solver++ 3M latent vs oracle")


def test_order_one_sampler_is_ddim_and_launches_match(mini):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    kw = dict(steps=5, shape=[1, 4, 16, 16], c_info=_cinfo(gi["c"], gi["u"]), verbose=False, eta=0.)
    with torch.no_grad():
        Sd, Sp = DDIMSampler(net), DPMSolverSampler(net, order=1)
        ref, _ = Sd.sample(x_info={"type": "image", "xt": gi["xT"]}, **kw)
        out, _ = Sp.sample(x_info={"type": "image", "xt": gi["xT"]}, **kw)
    out, ref = out.float().cpu().flatten(), ref.float().cpu().flatten()
    cos = torch.nn.functional.cosine_similarity(out, ref, dim=0).item()
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    print(f"[dpm] order 1 vs DDIMSampler, 5 steps: cos {cos:.8f}, max|err| {err:.3g} of max|ref|")
    assert cos >= 0.9999 and err <= 1e-2
    print(f"[dpm] launches per step: DDIM {Sd.last_step_launches}, DPM-Solver++ {Sp.last_step_launches}")
    assert Sp.last_step_launches == Sd.last_step_launches > 0


def test_graph_equals_eager_and_is_reusable(mini):
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    args = dict(steps=6, shape=[2, 4, 16, 16], verbose=False, eta=0.)
    g = torch.Generator().manual_seed(3)
    xT = torch.randn(2, 4, 16, 16, generator=g)
    c, u = torch.randn(2, 77, 768, generator=g).to(DEV), torch.randn(2, 77, 768, generator=g).to(DEV)

    def run(S, cc=c):
        with torch.no_grad():
            return S.sample(x_info={"type": "image", "xt": xT.clone()},
                            c_info={"type": "text", "conditioning": cc, "unconditional_conditioning": u,
                                    "unconditional_guidance_scale": 5.0}, **args)[0]
    eager = run(DPMSolverSampler(net, order=3, use_cuda_graph=False))
    Sg = DPMSolverSampler(net, order=3, use_cuda_graph=True)
    g1, g2 = run(Sg), run(Sg)
    assert torch.equal(g1, g2), "graph replay must be deterministic"
    assert torch.equal(eager, g1), "graph path must be bit-identical to the eager path"
    c2 = torch.randn(2, 77, 768, generator=g).to(DEV)
    g3 = run(Sg, c2)
    e3 = run(DPMSolverSampler(net, order=3, use_cuda_graph=False), c2)
    assert torch.equal(e3, g3), "replay-only path with a refreshed context must equal the eager path"
    with torch.no_grad():
        net.apply_model({"type": "image", "x": xT.to(DEV)}, torch.tensor([5, 5], device=DEV), {"type": "text", "c": c2})
    g4 = run(Sg)
    assert torch.equal(eager, g4), "graph must be rebuilt when the K / V^T buffers it captured were replaced"
    # another order on the same sampler: a new key, a new graph, the eager result of that order
    Sg.order = 2
    assert torch.equal(run(Sg), run(DPMSolverSampler(net, order=2, use_cuda_graph=False)))
