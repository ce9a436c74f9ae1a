"""Every sampling mode on every kind of walk, on the mini UNet against its oracle fed the draws the device used.

The modes (inpainting with a soft mask, also from the img2img start; a walk from an inversion with a mask; two regions with
bootstrapping; circular windows with an inpainting mask; SAG, also with inpainting; Prompt-to-Prompt replace with a local blend)
each meet the walks: the stochastic DPM-Solver++ (2M at eta 1 on the uniform and trailing grids, 3M at eta 0.5 on the Karras
grid), DPM-Solver++ 2M on the Karras grid, DDIM on the trailing grid, and the eager stochastic DDIM (eta 1, temperature 0.8).
The kernels are checked per element elsewhere; what these tests see is how the step graph wires a mode into a walk: which grid a
mode's per-step table is built on, whether the walk's noise reaches the CFG duplicate of the latent, and that windows and regions
add the noise once on the canvas.

Draws read back from the device: the SDE noise through test_dpm_sde_gpu.draws with the walk's key, the inpainting blend's through
vdb_inpaint_noise_f32, the bootstrap's through vdb_region_noise_f32, and the stochastic DDIM's by recording what
lib.model_zoo.ddim.noise_like returned.  Then bit-for-bit invariants under the SDE, the Karras grid shorter than its steps, and
the per-step tables the modes build (inpainting blend rows, SAG rows, region bootstrap rows) read back from the device against
rows built from the grid."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import dpm_sde_oracle as G
from oracle import edit_oracle as E
from oracle import inpaint_oracle as I
from oracle import panorama_oracle as P
from oracle import prompt_edit_oracle as PE
from oracle import regions_oracle as R
from oracle import sag_oracle as SG
from oracle import vd_oracle as O
from test_dpm_sde_gpu import draws
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
AC = O.ddpm_schedule(1000)["alphas_cumprod"]
STEPS = 8
# name -> (sampler kind, order, eta, grid, temperature)
WALKS = {"sde2-eta1-uniform": ("sde", 2, 1.0, "uniform", 1.0), "sde3-eta0.5-karras": ("sde", 3, 0.5, "karras", 1.0),
         "sde2-eta1-trailing": ("sde", 2, 1.0, "trailing", 1.0), "dpm2-karras": ("dpm", 2, 0.0, "karras", 1.0),
         "ddim-trailing": ("ddim", 1, 0.0, "trailing", 1.0), "ddim-eta1-t0.8-uniform": ("ddim", 1, 1.0, "uniform", 0.8)}
MODES = ["inpaint", "inpaint_img2img", "inversion", "regions", "windows", "sag", "sag_inpaint", "prompt_edit"]
# CFG scale of the mode cases: a walk from pure noise on the random-weight mini UNet amplifies bf16 rounding, the more so on the
# grids that start at t = 999 (at 7.5 the latent reaches ~100 in 8 steps); test_prompt_edit_gpu walks at 3 for the same reason
SCALE = 3.0
# SAG's mask is mass > 1 on a 3 x 3 mid map, so one cell that lands on the other side of the threshold on the device changes a
# ninth of the guidance.  At the last step the device's mass differs from the oracle's by 2e-3 - 1e-2 (mostly about 5e-3) on an
# H100, so each (mode, walk) takes, among input seeds 0 - 5, the one whose oracle masses stay farthest from 1 (>= 3.5e-3 on every
# step), and the test asserts that margin.  Over those 72 seeds the 4 that missed the bound all had margins below 2e-3 and a
# last-step mass 3e-2 - 5e-2 off, on three different walks: mask flips, not a walk's wiring, which would fail every seed.
SAG_SEEDS = {("sag", "sde2-eta1-uniform"): 3, ("sag", "sde3-eta0.5-karras"): 1, ("sag", "sde2-eta1-trailing"): 1,
             ("sag", "dpm2-karras"): 2, ("sag", "ddim-trailing"): 4, ("sag", "ddim-eta1-t0.8-uniform"): 5,
             ("sag_inpaint", "sde2-eta1-uniform"): 2, ("sag_inpaint", "sde3-eta0.5-karras"): 3,
             ("sag_inpaint", "sde2-eta1-trailing"): 2, ("sag_inpaint", "dpm2-karras"): 1, ("sag_inpaint", "ddim-trailing"): 5,
             ("sag_inpaint", "ddim-eta1-t0.8-uniform"): 0}
SAG_MARGIN = 3e-3


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=SCALE, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _sampler(net, walk, steps=STEPS, **kw):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler
    kind, order, _, grid, _ = walk
    if kind == "ddim":
        return DDIMSampler(net, grid=grid, **kw)
    return (DPMSolverSDESampler if kind == "sde" else DPMSolverSampler)(net, order=order, grid=grid, **kw)


@contextlib.contextmanager
def _recorded_ddim_noise():
    """what the eager stochastic DDIM loop drew (noise_like, NHWC), in walk order"""
    from lib.model_zoo import ddim
    rec, orig = [], ddim.noise_like

    def wrapped(x, repeat=False):
        z = orig(x, repeat)
        rec.append(z.clone())
        return z
    ddim.noise_like = wrapped
    try:
        yield rec
    finally:
        ddim.noise_like = orig


@contextlib.contextmanager
def _q_sample_noise(net, noise):
    """inject the img2img start's draw"""
    orig = net.q_sample
    net.q_sample = lambda x_start, t, noise_=None: orig(x_start, t, noise=noise.to(x_start.device).expand_as(x_start))
    try:
        yield
    finally:
        net.q_sample = orig


def _nchw(z, shape):
    bs, C, H, W = shape
    return z.reshape(bs, H, W, C).permute(0, 3, 1, 2).double().cpu().numpy()


def _run(S, walk, x_info, cl, shape, steps=STEPS, seed=0):
    """-> (latent, the walk's noise(i) in NCHW fp64 for the oracle, or None)"""
    kind, _, eta, _, temp = walk
    kw = dict(steps=steps, shape=shape, x_info=x_info, verbose=False, eta=eta, temperature=temp)
    torch.manual_seed(seed)
    with _recorded_ddim_noise() as rec, torch.no_grad():
        x = (S.sample_multicontext(c_info_list=cl, **kw) if len(cl) > 1 else S.sample(c_info=cl[0], **kw))[0]
    if eta == 0:
        return x, None
    if kind == "ddim":
        total = len(rec)
        return x, lambda i: temp * _nchw(rec[total - 1 - i], shape)
    key, n = S._st["sde_key"].clone(), int(np.prod(shape))
    # the oracle reads the draws back through the kernel, so it cannot see a counter that ignores the step: check that here
    top = len(S.ddim_timesteps) - 1
    assert (draws(key, top, n) != draws(key, top - 1, n)).float().mean().item() > 0.99, "the SDE draws differ from step to step"
    return x, lambda i: _nchw(draws(key, i, n), shape)


def _inpaint_noise(S, shape):
    from vdb200 import ops
    seed, n = S._st["seed"].clone(), int(np.prod(shape))
    return lambda i: torch.from_numpy(_nchw(ops.inpaint_noise(seed, _idx(i), n), shape)).float()


def _oracle_kw(walk):
    kind, order, eta, grid, _ = walk
    return dict(sampler="ddim" if kind == "ddim" else "dpmpp", order=order, grid_name=grid, eta=eta, model_channels=64)


def _mode_case(mode, net, sd, gi, walk, multi=False, seed=None, graph=True, oracle=True):
    """Run `mode` on `walk` on the device (on the captured step graph, or eager) and, with `oracle`, its oracle -> (latent,
    oracle latent or None, the oracle masses' least distance from SAG's threshold or None).  seed: of the inputs."""
    from lib.model_zoo import panorama
    from lib.model_zoo.regions import Region, Regions
    from lib.model_zoo.sag import SelfAttentionGuidance
    g = torch.Generator().manual_seed(101 + MODES.index(mode) if seed is None else seed)
    bs, C = 1, 4
    H, W = {"windows": (16, 32), "sag": (24, 24), "sag_inpaint": (24, 24)}.get(mode, (16, 16))
    shape = [bs, C, H, W]
    okw = dict(_oracle_kw(walk), scale=SCALE)
    if multi:
        conds = [gi["c"], torch.randn(bs, 257, 768, generator=g) * 0.5]
        unconds = [gi["u"], torch.zeros(bs, 257, 768)]
        cl = [_cinfo(conds[0], unconds[0], ratio=0.7), _cinfo(conds[1], unconds[1], typ="image", ratio=0.3)]
        okw.update(c_types=("text", "image"), ratios=[0.7, 0.3])
    else:
        conds, unconds = [gi["c"]], [gi["u"]]
        cl = [_cinfo(gi["c"], gi["u"])]
    xT = torch.randn(shape, generator=g)
    x0 = torch.randn(shape, generator=g) * 0.8
    soft = torch.rand(1, 1, H, W, generator=g)
    S = _sampler(net, walk, use_cuda_graph=graph)

    if mode in ("inpaint", "inpaint_img2img"):
        x_info = {"type": "image", "xt": xT.to(DEV), "x0": x0.to(DEV), "inpaint_mask": soft.to(DEV)}
        k, start = None, torch.randn(shape, generator=g)
        if mode == "inpaint_img2img":      # (an 'xt' would take precedence over the img2img start)
            k = 5
            del x_info["xt"]
            x_info["x0_forward_timesteps"] = k
        with _q_sample_noise(net, start):
            x, noise = _run(S, walk, x_info, cl, shape)
        if not oracle:
            return x, None, None
        ref = I.sample(sd, xT, conds, unconds, STEPS, x0, soft, _inpaint_noise(S, shape), x0_forward_timesteps=k, x0_noise=start,
                       noise=noise, **okw)
        return x, ref, None

    if mode == "inversion":
        inv = _sampler(net, ("ddim", 1, 0.0, walk[3], 1.0)).invert(STEPS, x0.to(DEV), _cinfo(gi["c"], gi["u"], scale=1.0), k=5)
        traj = inv.trajectory.permute(0, 1, 4, 2, 3).double().cpu()
        x, noise = _run(S, walk, {"type": "image", "inversion": inv, "inpaint_mask": soft.to(DEV)}, cl, shape)
        if not oracle:
            return x, None, None
        own = E.invert(sd, x0, conds[:1], unconds[:1], STEPS, k=5, grid_name=walk[3], model_channels=64)
        _cmp(traj, own, cos_min=0.999, tol=0.05, what=f"inversion on the {walk[3]} grid vs oracle")
        return x, E.sample(sd, traj, conds, unconds, STEPS, mask=soft, noise=noise, **okw), None

    if mode == "regions":
        from vdb200 import ops
        masks = torch.zeros(2, 1, H, W)
        masks[0, :, :, :W // 2] = 1.0
        masks[1, :, H // 2:, W // 2:] = 1.0      # binary: DDIM's paper-form step is the eps average only for binary masks
        bgs = torch.randn(3, C, generator=g) * 0.5
        rconds = [[gi["c"] * 0.5] + conds[1:], [gi["u"] * 0.7] + conds[1:]]
        regs = Regions([Region(masks[r].to(DEV), [c.to(DEV) for c in rconds[r]] if multi else rconds[r][0].to(DEV))
                        for r in range(2)], bootstrap_steps=3, backgrounds=bgs.to(DEV))
        x, noise = _run(S, walk, {"type": "image", "xt": xT.to(DEV), "regions": regs}, cl, shape)
        seed, n = S._st["regions"].seed.clone(), int(np.prod(shape))
        if walk[0] == "sde":
            # the SDE key is drawn with the modes, the bootstrap key at the walk's start after them
            torch.manual_seed(0)
            keys = torch.randint(-2 ** 63, 2 ** 63 - 1, (2,), dtype=torch.int64)
            assert int(S._st["sde_key"]) == int(keys[0]) and int(seed) == int(keys[1])
        if not oracle:
            return x, None, None
        boot = lambda i: ops.region_noise(seed, _idx(i), n, 2, bs, 3)
        ref = R.sample(sd, xT, conds, unconds, rconds, masks.numpy().astype(np.float64), STEPS, bootstrap_steps=3,
                       backgrounds=bgs.numpy(), pick_fn=lambda i: boot(i)[1].cpu().numpy(), z_fn=lambda i: _nchw(boot(i)[0], shape),
                       noise=noise, **okw)
        return x, ref, None

    if mode == "windows":
        x_info = {"type": "image", "xt": xT.to(DEV), "x0": x0.to(DEV), "inpaint_mask": soft.to(DEV),
                  "windows": panorama.Windows(16, 8, circular=True)}
        x, noise = _run(S, walk, x_info, cl, shape)
        if not oracle:
            return x, None, None
        ref = P.sample(sd, xT, conds, unconds, STEPS, 16, 8, circular=True, x0=x0, mask=soft, noise_fn=_inpaint_noise(S, shape),
                       noise=noise, **okw)
        return x, ref, None

    if mode in ("sag", "sag_inpaint"):
        x_info = {"type": "image", "xt": xT.to(DEV), "sag": SelfAttentionGuidance(0.75)}
        if mode == "sag_inpaint":
            x_info.update(x0=x0.to(DEV), inpaint_mask=soft.to(DEV))
        x, noise = _run(S, walk, x_info, cl, shape)
        if not oracle:
            return x, None, None
        masses = []
        ref = SG.sample(sd, xT, conds, unconds, STEPS, 0.75, masses=masses, noise=noise,
                        **(dict(x0=x0, mask=soft, noise_fn=_inpaint_noise(S, shape)) if mode == "sag_inpaint" else {}), **okw)
        dev_last = S._st["sag_mass"].double().cpu()         # the mass of the walk's last step
        return x, ref, ((torch.cat([v.flatten() for v in masses]) - 1).abs().min().item(),
                        (dev_last - masses[-1]).abs().max().item())

    assert mode == "prompt_edit"
    from test_prompt_edit_gpu import _contexts, _edit
    n = 3
    ed, comp, c = _edit("replace", True)
    pconds, punconds, pkw, cl_fn = _contexts(n, multi, g)
    xt = torch.randn(1, C, H, W, generator=g).expand(n, C, H, W).contiguous()
    x, noise = _run(S, walk, {"type": "image", "xt": xt.to(DEV)}, cl_fn(ed), [n, C, H, W])
    if not oracle:
        return x, None, None
    T = len(S.ddim_timesteps)
    ctl = PE.P2P(n, "replace", T, ed.cross_steps, ed.self_steps, c, H, W, w=ed.blend, threshold=ed.threshold, **comp)
    okw.update(pkw)
    ref = PE.sample(sd, ctl, xt, pconds, punconds, STEPS, noise=noise, **okw)
    return x, ref, None


@pytest.mark.parametrize("walk", list(WALKS))
@pytest.mark.parametrize("mode", MODES)
def test_mode_on_walk_vs_oracle(mini, mode, walk):
    net, sd, gi = mini
    x, ref, sag = _mode_case(mode, net, sd, gi, WALKS[walk], seed=SAG_SEEDS.get((mode, walk)))
    if sag is not None:
        margin, dmass = sag
        print(f"[modes] {mode} on {walk}: oracle masses min |mass - 1| {margin:.2e}, last-step device mass off by {dmass:.2e}")
        assert margin >= SAG_MARGIN, "a mass this close to the threshold could flip the mask: pick another seed"
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"{mode} on {walk} vs oracle")


@pytest.mark.parametrize("mode", ["inpaint", "regions", "prompt_edit"])
def test_multicontext_mode_vs_oracle(mini, mode):
    net, sd, gi = mini
    x, ref, _ = _mode_case(mode, net, sd, gi, WALKS["sde2-eta1-uniform"], multi=True)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"dual-context {mode} on sde2-eta1-uniform vs oracle")


# ---- bit-for-bit invariants under the SDE (eta 1, Karras grid) -----------------------------------------------------------------
SDE_KARRAS = ("sde", 2, 1.0, "karras", 1.0)


def test_inpaint_mask_extremes(mini):
    net, _, gi = mini
    g = torch.Generator().manual_seed(7)
    shape = [2, 4, 16, 16]
    xT, x0 = torch.randn(shape, generator=g).to(DEV), (torch.randn(shape, generator=g) * 0.8).to(DEV)
    c, u = gi["c"].repeat(2, 1, 1), gi["u"].repeat(2, 1, 1)
    info = lambda m: {"type": "image", "xt": xT.clone(), "x0": x0, "inpaint_mask": torch.full((1, 1, 16, 16), m, device=DEV)}
    keep, _ = _run(_sampler(net, SDE_KARRAS), SDE_KARRAS, info(0.0), [_cinfo(c, u)], shape, seed=3)
    assert torch.equal(keep, x0), "mask 0 keeps x0"
    gen, _ = _run(_sampler(net, SDE_KARRAS), SDE_KARRAS, info(1.0), [_cinfo(c, u)], shape, seed=3)
    # the inpainting key is drawn first, then the SDE key: a plain walk after one extra draw has the same SDE key
    torch.manual_seed(3)
    torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)
    with torch.no_grad():
        plain = _sampler(net, SDE_KARRAS).sample(steps=STEPS, shape=shape, x_info={"type": "image", "xt": xT.clone()},
                                                 c_info=_cinfo(c, u), verbose=False, eta=1.0)[0]
    assert torch.equal(gen, plain), "mask 1 is the plain SDE walk"


def test_prompt_edit_source_row_and_one_window(mini):
    from lib.model_zoo import panorama
    from test_prompt_edit_gpu import _contexts, _edit
    net, _, gi = mini
    g = torch.Generator().manual_seed(9)
    n, shape = 3, [3, 4, 16, 16]
    ed, _, _ = _edit("replace", True)
    _, _, _, cl_fn = _contexts(n, False, g)
    xt = torch.randn(1, 4, 16, 16, generator=g).expand(*shape).contiguous().to(DEV)
    edited, _ = _run(_sampler(net, SDE_KARRAS), SDE_KARRAS, {"type": "image", "xt": xt}, cl_fn(ed), shape, seed=4)
    plain, _ = _run(_sampler(net, SDE_KARRAS), SDE_KARRAS, {"type": "image", "xt": xt}, cl_fn(None), shape, seed=4)
    assert torch.equal(edited[0], plain[0]), "the source row is the unedited batch's row 0"
    assert not torch.equal(edited[1:], plain[1:])
    one, _ = _run(_sampler(net, SDE_KARRAS), SDE_KARRAS, {"type": "image", "xt": xt, "windows": panorama.Windows(16, 16)},
                  cl_fn(None), shape, seed=4)
    assert torch.equal(one, plain), "one window equal to the canvas is the unwindowed walk"


@pytest.mark.parametrize("mode", MODES)
def test_graph_equals_eager(mini, mode):
    net, sd, gi = mini
    outs = [_mode_case(mode, net, sd, gi, SDE_KARRAS, graph=graph, oracle=False)[0] for graph in (True, False)]
    assert torch.equal(outs[0], outs[1]), mode


# ---- the Karras grid shorter than its steps ------------------------------------------------------------------------------------
def test_prompt_edit_windows_span_the_short_karras_walk(mini):
    """68 Karras steps walk fewer grid points: the edit's windows are fractions of the walk's length"""
    net, sd, gi = mini
    walk = ("sde", 2, 1.0, "karras", 1.0)
    steps = 68
    T = len(G.grid("karras", steps, AC.numpy()))
    assert T < steps
    from test_prompt_edit_gpu import _contexts, _edit
    g = torch.Generator().manual_seed(13)
    n, C, H, W = 3, 4, 16, 16
    ed, comp, c = _edit("replace", True)
    pconds, punconds, pkw, cl_fn = _contexts(n, False, g)
    xt = torch.randn(1, C, H, W, generator=g).expand(n, C, H, W).contiguous()
    S = _sampler(net, walk)
    x, noise = _run(S, walk, {"type": "image", "xt": xt.to(DEV)}, cl_fn(ed), [n, C, H, W], steps=steps)
    assert len(S.ddim_timesteps) == T
    # the edit's tables on the device are those of a walk of T steps, not of `steps`
    es, want = S._st["prompt_edit"], ed.tables(T, True)
    for name, dev in (("cross", es.cross), ("self", es.selfm), ("flags", es.flags)):
        assert np.array_equal(dev[:T].cpu().numpy(), want[name]), name
    assert not np.array_equal(es.cross[:T].cpu().numpy(), ed.tables(steps, True)["cross"][:T])
    ctl = PE.P2P(n, "replace", T, ed.cross_steps, ed.self_steps, c, H, W, w=ed.blend, threshold=ed.threshold, **comp)
    ref = PE.sample(sd, ctl, xt, pconds, punconds, steps, scale=SCALE, noise=noise, **_oracle_kw(walk), **pkw)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"prompt edit on the {T}-point Karras walk of {steps} steps vs oracle")


# ---- the modes' per-step tables are built on the walk's grid -----------------------------------------------------------------
@pytest.mark.parametrize("grid", ["karras", "trailing"])
def test_step_tables_follow_the_grid(mini, grid):
    """The inpainting blend rows, SAG's rows and the regions' bootstrap rows, read back from the device after a walk, against rows
    built from the grid (inpaint_oracle.blend_rows; {sqrt(ac_t), sqrt(1 - ac_t)} at each grid point)."""
    from lib.model_zoo.regions import Region, Regions
    from lib.model_zoo.sag import SelfAttentionGuidance
    net, _, gi = mini
    walk = ("sde", 2, 1.0, grid, 1.0)
    ts = G.grid(grid, STEPS, AC.numpy())
    n = len(ts)
    a = AC.numpy().astype(np.float64)[ts]
    at = np.stack([np.sqrt(a), np.sqrt(1.0 - a)], axis=1)
    H = W = 24
    x_info = {"type": "image", "xt": torch.zeros(1, 4, H, W, device=DEV), "x0": torch.zeros(1, 4, H, W, device=DEV),
              "inpaint_mask": torch.full((1, 1, H, W), 0.5, device=DEV), "sag": SelfAttentionGuidance(0.75)}
    S = _sampler(net, walk)
    _run(S, walk, x_info, [_cinfo(gi["c"], gi["u"])], [1, 4, H, W])
    assert np.array_equal(S.ddim_timesteps, ts)
    torch.testing.assert_close(S._st["blend"][:n].cpu(), torch.from_numpy(I.blend_rows(AC.numpy(), ts)).float(), rtol=1e-6, atol=0)
    torch.testing.assert_close(S._st["sag_tab"][:n].cpu(), torch.from_numpy(at).float(), rtol=1e-6, atol=0)
    boot = 3
    regs = Regions([Region(torch.ones(1, H, W, device=DEV), gi["c"].to(DEV))], bootstrap_steps=boot,
                   backgrounds=torch.zeros(2, 4, device=DEV))
    S = _sampler(net, walk)
    _run(S, walk, {"type": "image", "xt": torch.zeros(1, 4, H, W, device=DEV), "regions": regs}, [_cinfo(gi["c"], gi["u"])],
         [1, 4, H, W])
    rows = np.zeros((n, 4))
    rows[:, 0] = np.arange(n) >= n - boot
    rows[:, 1:3] = at
    torch.testing.assert_close(S._st["regions"].rows[:n].cpu(), torch.from_numpy(rows).float(), rtol=1e-6, atol=0)
