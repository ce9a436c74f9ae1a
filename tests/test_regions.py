"""Region prompts, CPU side (lib/model_zoo/regions.py): Region / Regions validation and every refusal of the samplers with its
exception type, the weight rule (m_0 and D) on a dense grid of fp32 mask values, the bootstrap step rows under DDIM, DPM-Solver++
and an img2img start, the argument checks of the C entry points, and the oracle (oracle/regions_oracle.py): its paper-form DDIM
step against the eps average for binary masks, and all-zero masks reducing it to the plain (windowed) walk."""
import types

import numpy as np
import pytest
import torch

from oracle import dpm_solver_oracle as D
from oracle import panorama_oracle as P
from oracle import regions_oracle as G
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def _cinfo(bs=1, L=77, **kw):
    return dict({"type": "text", "conditioning": torch.zeros(bs, L, 768), "unconditional_conditioning": torch.zeros(bs, L, 768),
                 "unconditional_guidance_scale": 7.5}, **kw)


def _samplers():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return [DDIMSampler(_fake_model()), DPMSolverSampler(_fake_model())]


def _regions(R=2, bs=1, H=16, W=24, multi=False, **kw):
    from lib.model_zoo.regions import Region, Regions
    c = torch.zeros(bs, 77, 768)
    return Regions([Region(torch.zeros(1, H, W), [c, c] if multi else c) for _ in range(R)], **kw)


def test_region_and_regions_refusals():
    from lib.model_zoo.regions import REGIONS_MAX, Region, Regions
    c, m = torch.zeros(1, 77, 768), torch.zeros(1, 16, 24)
    for bad in (np.zeros((1, 16, 24), np.float32), torch.zeros(1, 16, 24, dtype=torch.float64), None):
        with pytest.raises(ValueError, match="fp32 tensor"):
            Region(bad, c)
    for bad in (None, [], [c, None], np.zeros((1, 77, 768))):
        with pytest.raises(ValueError, match="conditioning"):
            Region(m, bad)
    assert REGIONS_MAX == 8
    for n in (0, 9):
        with pytest.raises(ValueError, match="1 to 8 regions"):
            Regions([Region(m, c)] * n)
    Regions([Region(m, c)] * 8)
    with pytest.raises(ValueError, match="every entry"):
        Regions([Region(m, c), (m, c)])
    for bad in (-1, 1.0, True, "2"):
        with pytest.raises(ValueError, match="bootstrap_steps"):
            Regions([Region(m, c)], bootstrap_steps=bad)
    with pytest.raises(ValueError, match="needs backgrounds"):
        Regions([Region(m, c)], bootstrap_steps=3)
    for bad in (torch.zeros(4), torch.zeros(0, 4), torch.full((2, 4), float("nan")), np.zeros((2, 4))):
        with pytest.raises(ValueError, match="backgrounds must be"):
            Regions([Region(m, c)], bootstrap_steps=3, backgrounds=bad)
    Regions([Region(m, c)], bootstrap_steps=3, backgrounds=torch.zeros(2, 4))


@pytest.mark.parametrize("multi", [False, True])
def test_sampler_refusals(multi):
    """Every refusal is raised before any device work (the fake model is on the CPU, where a call that passed them would raise
    RuntimeError instead), with its type; nothing is drawn from torch's CPU generator on the way."""
    from lib.model_zoo.panorama import Windows
    from lib.model_zoo.regions import Region, Regions
    bs, H, W = 2, 16, 24
    shape = [bs, 4, H, W]
    c = torch.zeros(bs, 77, 768)
    cond = [c, torch.zeros(bs, 257, 768)] if multi else c

    def run(S, x_info, shape=shape, **ci):
        if multi:
            cl = [_cinfo(bs, **ci), _cinfo(bs, 257, type="image")]
            return S.sample_multicontext(steps=5, shape=shape, x_info=x_info, c_info_list=cl, verbose=False)
        return S.sample(steps=5, shape=shape, x_info=x_info, c_info=_cinfo(bs, **ci), verbose=False)

    def regs(mask=None, conds=None, width=W, **kw):
        return Regions([Region(torch.zeros(1, H, width) if mask is None else mask, cond if conds is None else conds)], **kw)

    bg = torch.zeros(3, 4)
    for S in _samplers():
        torch.manual_seed(0)
        state = torch.get_rng_state()
        refusals = [
            (ValueError, "regions.Regions", {"regions": [Region(torch.zeros(1, H, W), cond)]}, shape, {}),
            (ValueError, "text latent", {"regions": regs()}, [bs, 768], {}),
            (ValueError, "mask expected", {"regions": regs(torch.zeros(1, 1, H, W))}, shape, {}),
            (ValueError, "mask expected", {"regions": regs(torch.zeros(3, H, W))}, shape, {}),
            (ValueError, "mask expected", {"regions": regs(torch.zeros(1, H, W + 8))}, shape, {}),
            (ValueError, "mask expected", {"regions": regs(torch.zeros(1, 4 * H, 4 * W))}, shape, {}),
            (ValueError, "lie in \\[0, 1\\]", {"regions": regs(torch.full((1, H, W), 1.5))}, shape, {}),
            (ValueError, "lie in \\[0, 1\\]", {"regions": regs(torch.full((bs, 8 * H, 8 * W), -0.25))}, shape, {}),
            (ValueError, "lie in \\[0, 1\\]", {"regions": regs(torch.full((1, H, W), float("nan")))}, shape, {}),
            (ValueError, "conditioning 0 expected", {"regions": regs(conds=[torch.zeros(bs, 70, 768)] + ([cond[1]] if multi else []))},
             shape, {}),
            (ValueError, "conditioning tensors for", {"regions": regs(conds=[c, c, c])}, shape, {}),
            (ValueError, "bootstrap_steps must lie in", {"regions": regs(bootstrap_steps=6, backgrounds=bg)}, shape, {}),
            (ValueError, "backgrounds expected", {"regions": regs(bootstrap_steps=2, backgrounds=torch.zeros(3, 5))}, shape, {}),
            (ValueError, "panorama.Windows", {"regions": regs(), "windows": (16, 8)}, shape, {}),
            (ValueError, "multiple of the stride", {"regions": regs(width=40), "windows": Windows(16, 16, circular=True)},
             [bs, 4, H, 40], {}),
            (NotImplementedError, "regions with prompt_edit", {"regions": regs()}, shape, {"prompt_edit": object()}),
            (NotImplementedError, "regions cannot sample from an inversion", {"regions": regs(), "inversion": object()}, shape, {}),
        ]
        for exc, match, x_info, shp, ci in refusals:
            with pytest.raises(exc, match=match):
                run(S, dict({"type": "image"}, **x_info), shape=shp, **ci)
        # valid inputs pass the checks and reach the device check: latent / pixel / per-item / soft masks, bootstrapping, windows
        # (circular too), the img2img start, inpainting
        gen = torch.Generator().manual_seed(1)
        pix, soft = torch.rand(bs, 8 * H, 8 * W, generator=gen), torch.rand(1, H, W, generator=gen)
        for x_info in ({"regions": regs()}, {"regions": regs(pix)}, {"regions": regs(soft)},
                       {"regions": regs(bootstrap_steps=5, backgrounds=bg)},
                       {"regions": regs(), "windows": Windows(16, 8)}, {"regions": regs(), "windows": Windows(8, 8, circular=True)},
                       {"regions": regs(), "x0": torch.zeros(1, 4, H, W), "x0_forward_timesteps": 3}):
            with pytest.raises(RuntimeError, match="no CPU path"):
                run(S, dict({"type": "image"}, **x_info))
        assert torch.equal(torch.get_rng_state(), state), "the key is drawn after the device check, and only when bootstrapping"
        with pytest.raises(RuntimeError, match="no CPU path"):      # outpainting with regions (inpainting draws its own key)
            run(S, {"type": "image", "regions": regs(), "x0": torch.zeros(1, 4, H, W), "inpaint_mask": torch.ones(1, 1, H, W)})


def test_plms_and_the_single_step_api_refuse_regions():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.plms import PLMSSampler
    S = PLMSSampler(_fake_model())
    with pytest.raises(NotImplementedError, match="PLMSSampler has no region prompts"):
        S.sample(steps=5, shape=[1, 4, 16, 24], x_info={"type": "image", "regions": _regions()}, c_info=_cinfo(), verbose=False)
    S = DDIMSampler(_fake_model())
    S.make_schedule(5, verbose=False)
    with pytest.raises(NotImplementedError, match="region prompts run inside the sampler's walk"):
        S.p_sample_ddim({"type": "image", "x": torch.zeros(1, 4, 16, 24), "regions": _regions()}, _cinfo(),
                        torch.zeros(1, dtype=torch.long), 0)


def test_regions_take_the_windows():
    """Windows given with regions select no window walk of their own: the region mode reads the layout.  Windows alone select the
    same mode with no regions (R = 0), in chunks of WINDOWS_PER_CHUNK windows."""
    from lib.model_zoo.ddim import TAKES, DDIMSampler
    from lib.model_zoo.panorama import WINDOWS_PER_CHUNK, Windows
    from lib.model_zoo.regions import RegionPrompts
    assert TAKES["regions"] == ("windows",)
    S = DDIMSampler(_fake_model())
    S.make_schedule(5, verbose=False)
    modes = S._modes("sample", {"type": "image", "regions": _regions(W=40), "windows": Windows(16, 8)}, [1, 4, 16, 40], [_cinfo()])
    assert [type(m) for m in modes] == [RegionPrompts]
    m = modes[0]
    assert m.lay.nwin == 4 and m.per == 2 and m.chunks == [(0, 2), (2, 2)], "8 // (R + 1) windows per chunk"
    m = S._modes("sample", {"type": "image", "regions": _regions(R=8)}, [1, 4, 16, 24], [_cinfo()])[0]
    assert (m.lay.h, m.lay.w, m.lay.nwin, m.per) == (16, 24, 1, 1), "no windows: one window, the canvas"
    modes = S._modes("sample", {"type": "image", "windows": Windows(64, 8)}, [1, 4, 64, 256], [_cinfo()])
    assert [type(m) for m in modes] == [RegionPrompts]
    m = modes[0]
    assert m.R == 0 and not m.boot and m.per == WINDOWS_PER_CHUNK == 8
    assert m.lay.nwin == 25 and m.chunks == [(0, 8), (8, 8), (16, 8), (24, 1)]


def test_the_weight_rule_on_a_dense_grid():
    """m_0 = max(0, 1 - S) and D = m_0 + S in fp32: D is S when S >= 1, and 1 up to one rounding otherwise, so it is never
    below 1 - 2^-24 and never 0, for every combination of mask values on a dense grid of fp32 values in [0, 1]."""
    from lib.model_zoo.regions import weights
    u = np.float32(2.0 ** -24)
    special = np.array([0, 1, u, 2 * u, 1 - u, 1 - 2 * u, 0.5, 0.5 - u, 0.5 + u, 1 / 3, 2 / 3, 1e-30, 1e-8, 1 - 1e-7, 0.1, 0.9],
                       dtype=np.float32)
    grid = np.concatenate([special, np.linspace(0, 1, 257, dtype=np.float32),
                           np.random.default_rng(0).random(200).astype(np.float32)])
    for R, vals in ((1, np.concatenate([grid, np.nextafter(np.float32(1), np.float32(0)) - np.arange(64, dtype=np.float32) * u,
                                        np.arange(64, dtype=np.float32) * u])),
                    (2, grid), (3, grid[:48]), (8, special[:4])):
        combos = np.stack(np.meshgrid(*[vals] * R, indexing="ij")).reshape(R, -1)
        m0, Dn = weights(combos)
        S = combos[0].copy()
        for r in range(1, R):
            S = (S + combos[r]).astype(np.float32)
        assert m0.dtype == np.float32 and Dn.dtype == np.float32
        assert np.all(m0 >= 0) and np.all(m0 <= 1)
        assert np.all(Dn > 0) and np.all(Dn >= 1 - u), R
        assert np.array_equal(Dn[S >= 1], S[S >= 1])
        assert np.all(np.abs(Dn[S < 1].astype(np.float64) - 1.0) <= 2.0 ** -24), R
    # a hard mask, and all-zero masks: the selected weight is 1 and D is 1 exactly
    m0, Dn = weights(np.array([[0, 1, 0], [1, 0, 0]], dtype=np.float32))
    assert np.array_equal(m0, [0, 0, 1]) and np.array_equal(Dn, [1, 1, 1])


@pytest.mark.parametrize("kind,steps,k,boot", [("ddim", 50, None, 10), ("dpm", 20, None, 20), ("ddim", 10, 6, 3), ("dpm", 25, 9, 0),
                                               ("ddim", 5, None, 0)])
def test_step_rows(kind, steps, k, boot):
    """{on, sqrt(ac_t), sqrt(1 - ac_t), 0} of the latent entering each step, indexed by the grid index; on for the first `boot`
    steps walked, from the top of the walk (an img2img start walks the first k grid points)."""
    from lib.model_zoo.regions import step_rows
    S = _samplers()[kind == "dpm"]
    S.make_schedule(steps, verbose=False)
    ts = O.make_ddim_timesteps(steps)
    total = len(ts) if k is None else k
    rows = step_rows(S.ddim_alphas, total, boot)
    assert rows.dtype == np.float32 and rows.shape == (total, 4)
    ac = AC.numpy().astype(np.float64)[ts[:total]]
    assert np.array_equal(rows[:, 1], np.sqrt(ac).astype(np.float32))
    assert np.array_equal(rows[:, 2], np.sqrt(1.0 - ac).astype(np.float32))
    assert np.all(rows[:, 3] == 0)
    walked = list(range(total - 1, -1, -1))
    assert [bool(rows[i, 0]) for i in walked] == [n < boot for n in range(total)]


def test_entry_points_reject_bad_arguments_at_every_R_without_gpu():
    """vdb_region_gather_f32, vdb_region_merge_f32 and vdb_region_noise_f32 refuse null, misaligned, empty, out-of-range and
    overlapping arguments before any launch (the fake addresses are never dereferenced: every call fails its checks).  R = 0, a
    panorama's walk, needs no masks."""
    from vdb200._lib import lib
    bs, H, W, C, h, w, ny, nx, R = 2, 16, 40, 4, 16, 16, 1, 4, 2
    nin = bs * H * W * C
    ok = dict(x=0x1000000, bs=bs, H=H, W=W, C=C, oy=0x2000000, ox=0x2100000, ny=ny, nx=nx, h=h, w=w, first=0, k=nx, R=R, ub=1,
              masks=0x5000000, rows=0x5100000, idx=0x5200000, seed=0x5300000, bg=0x5400000, nb=3, noise=0x5500000,
              out=0x3000000, cy=0x2200000, cx=0x2300000, halves=2, z=0x6000000, picks=0x6100000, n=nin)

    def gather(**kw):
        a = dict(ok, **kw)
        return lib.vdb_region_gather_f32(a["x"], a["bs"], a["H"], a["W"], a["C"], a["oy"], a["ox"], a["ny"], a["nx"], a["h"],
                                         a["w"], a["first"], a["k"], a["R"], a["ub"], a["masks"], a["rows"], a["idx"], a["seed"],
                                         a["bg"], a["nb"], a["noise"], a["out"], None)

    def merge(**kw):
        a = dict(ok, **kw)
        return lib.vdb_region_merge_f32(a["x"], a["halves"], a["bs"], a["H"], a["W"], a["C"], a["oy"], a["ox"], a["cy"], a["cx"],
                                        a["ny"], a["nx"], a["h"], a["w"], a["first"], a["k"], a["R"], a["masks"], a["out"], None)

    def noise(**kw):
        a = dict(ok, **kw)
        return lib.vdb_region_noise_f32(a["seed"], a["idx"], a["n"], a["R"], a["bs"], a["nb"], a["z"], a["picks"], None)

    err = lambda: lib.vdb_last_error()
    before = lib.vdb_launch_count()
    for fn, what in ((gather, b"region_gather"), (merge, b"region_merge")):
        for key in ("x", "oy", "ox", "out") + (("cy", "cx", "masks") if fn is merge else ()):
            assert fn(**{key: None}) == 1 and what + b": null" in err(), key
        for key in ("bs", "H", "W", "C", "ny", "nx", "h", "w", "k"):
            for v in (0, -1):
                assert fn(**{key: v}) == 1 and b"empty" in err(), (key, v)
        assert fn(h=H + 1) == 1 and b"larger than the canvas" in err()
        assert fn(w=W + 8) == 1 and b"larger than the canvas" in err()
        for first, k in ((-1, 2), (3, 2), (0, 5), (4, 1)):
            assert fn(first=first, k=k) == 1 and b"outside the layout" in err(), (first, k)
        for key in ("oy", "ox"):
            assert fn(**{key: ok[key] + 2}) == 1 and b"4-byte aligned" in err(), key
        for bad in (-1, 9, 100):
            assert fn(R=bad) == 1 and b"R must be in [0, 8]" in err(), bad
        # R = 0 without masks passes the null checks and fails on the next refusal
        assert fn(R=0, masks=None, out=ok["out"] + 4) == 1 and b"16-byte aligned" in err()
    for ub in (2, -1, R + 2):
        assert gather(ub=ub) == 1 and b"u_blocks" in err(), ub
    for ub in (2, -1):
        assert gather(R=0, masks=None, ub=ub) == 1 and b"u_blocks must be 0, 1 or R + 1 = 1" in err(), ub
    for key in ("masks", "idx", "seed", "bg"):
        assert gather(**{key: None}) == 1 and b"rows needs" in err(), key
    assert gather(nb=0) == 1 and b"rows needs" in err()
    for key in ("x", "out", "noise"):
        assert gather(**{key: ok[key] + 4}) == 1 and b"16-byte aligned" in err(), key
    for key in ("masks", "rows", "bg", "idx"):
        assert gather(**{key: ok[key] + 2}) == 1 and b"aligned" in err(), key
    assert gather(seed=ok["seed"] + 4) == 1 and b"seed 8-byte" in err()
    for key in ("x", "out", "cx"):
        assert merge(**{key: ok[key] + 4}) == 1 and b"16-byte aligned" in err(), key
    for key in ("cy", "masks"):
        assert merge(**{key: ok[key] + 2}) == 1 and b"4-byte" in err(), key
    for v in (0, 3):
        assert merge(halves=v) == 1 and b"halves" in err(), v
    # overlaps: the batch against the canvas, the masks, the noise and the backgrounds (first and last shared float)
    nout = (1 + R + 1) * nx * bs * h * w * C
    for key, n in (("x", nin), ("masks", R * bs * H * W), ("noise", nin), ("bg", 3 * C)):
        a = ok[key]
        for addr in (a, a + 4 * (n - 4), a - 4 * (nout - 4)):
            assert gather(out=addr) == 1 and b"out overlaps" in err(), (key, addr)
    m_in, m_out = 2 * (R + 1) * nx * bs * h * w * C, 2 * bs * H * W * C
    for key, n in (("x", m_in), ("masks", R * bs * H * W)):
        a = ok[key]
        for addr in (a, a + 4 * (n - 4), a - 4 * (m_out - 4)):
            assert merge(out=addr) == 1 and b"overlaps out" in err(), (key, addr)
    for key in ("seed", "idx", "z", "picks"):
        assert noise(**{key: None}) == 1 and b"region_noise: null" in err(), key
    for key in ("n", "bs", "nb"):
        assert noise(**{key: 0}) == 1 and b"empty" in err(), key
    for bad in (0, 9):
        assert noise(R=bad) == 1 and b"R must be in [1, 8]" in err(), bad
    assert lib.vdb_launch_count() == before


# ---- the oracle on an analytic eps function ---------------------------------------------------------------------------------------
def _eps(i):
    """an eps that depends on the crop, the window, the region and the step, so views disagree"""
    return lambda xc, g, r: np.tanh(0.7 * xc) * (1.0 + 0.1 * g - 0.2 * r) + 0.03 * (g - 2) + 0.05 * r + 0.01 * i


def _binary_masks(R, bs, H, W, seed):
    g = np.random.default_rng(seed)
    lab = g.integers(0, R + 1, size=(bs, H, W))          # 0: background, r: region r
    m = np.stack([(lab == r).astype(np.float64) for r in range(1, R + 1)])
    m[:, :, :2, :2] = 1.0                                 # overlapping regions: S > 1 where they meet
    return m


@pytest.mark.parametrize("H,W,size,stride,circular,R,boot", [(16, 24, None, None, False, 2, False), (16, 24, None, None, False, 3, True),
                                                             (16, 40, 16, 8, False, 2, True), (16, 40, 16, 8, True, 1, False),
                                                             (24, 20, 16, 7, False, 4, True)])
def test_oracle_paper_form_equals_the_eps_average_for_binary_masks(H, W, size, stride, circular, R, boot):
    """With binary masks m_r x_r = m_r x, also under bootstrapping, so the mask-weighted per-view x_{t-1} is the update of the
    weighted eps average: in fp64 up to rounding."""
    sched = O.ddim_schedule(AC, 10)
    g = np.random.default_rng(H * W + R)
    bs, C = 2, 4
    x = g.standard_normal((bs, C, H, W))
    masks = _binary_masks(R, bs, H, W, H + R)
    h, w, wins = P.windows(H, W, max(H, W) if size is None else size, max(H, W) if stride is None else stride, circular)
    for i in (9, 4, 0):
        a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
        bt = (g.standard_normal((R, bs, C)), g.standard_normal((bs, C, H, W)), np.sqrt(a_t), np.sqrt(1 - a_t)) if boot else None
        paper = G.paper_step(x, _eps(i), masks, wins, h, w, a_t, a_prev, bt)
        via_eps = P.ddim_update(x, G.eps_average(x, _eps(i), masks, wins, h, w, bt), a_t, a_prev)
        assert np.abs(paper - via_eps).max() <= 1e-12 * np.abs(paper).max(), i
        # the regions disagree, so the result is not the background's walk
        bg_only = P.ddim_update(x, P.eps_average(x, lambda xc, gg: _eps(i)(xc, gg, 0), wins, h, w), a_t, a_prev)
        assert np.abs(paper - bg_only).max() > 1e-3
        x = paper


def test_oracle_soft_masks_with_bootstrap_differ_from_the_paper_form():
    """The docstring's caveat: with soft masks and bootstrapping the views' inputs differ inside the mask, so the eps average is a
    definition of its own, not the paper's x_{t-1} average (without bootstrapping the two agree for soft masks too)."""
    H, W, bs, C, R = 8, 8, 1, 4, 2
    g = np.random.default_rng(5)
    x = g.standard_normal((bs, C, H, W))
    masks = g.random((R, bs, H, W))
    h, w, wins = P.windows(H, W, 8, 8)
    a_t, a_prev = 0.3, 0.5
    bt = (g.standard_normal((R, bs, C)), g.standard_normal((bs, C, H, W)), np.sqrt(a_t), np.sqrt(1 - a_t))
    for boot, same in ((None, True), (bt, False)):
        paper = G.paper_step(x, _eps(3), masks, wins, h, w, a_t, a_prev, boot)
        via_eps = P.ddim_update(x, G.eps_average(x, _eps(3), masks, wins, h, w, boot), a_t, a_prev)
        assert (np.abs(paper - via_eps).max() <= 1e-12 * np.abs(paper).max()) == same


def test_oracle_all_zero_masks_are_the_plain_walk():
    """All-zero region masks: m_0 = 1 and D = 1, so the region walk is the plain (windowed) walk exactly, DDIM through the paper
    form and DPM-Solver++ through its eps average."""
    H, W, R = 16, 40, 3
    masks = np.zeros((R, 1, H, W))
    ts = O.make_ddim_timesteps(8)
    x = np.random.default_rng(1).standard_normal((1, 4, H, W))
    h, w, wins = P.windows(H, W, 16, 8)
    eps = lambda xv, i: np.tanh(0.7 * xv) + 0.01 * i
    for order in (1, 2):
        windowed = D.walk(x, lambda xv, i: P.eps_average(xv, lambda xc, g: eps(xc, i), wins, h, w), AC.numpy(), ts, order)
        regional = D.walk(x, lambda xv, i: G.eps_average(xv, lambda xc, g, r: eps(xc, i) + r, masks, wins, h, w), AC.numpy(),
                          ts, order)
        assert np.array_equal(windowed, regional), order
    sched = O.ddim_schedule(AC, 8)
    xp, xr = x, x
    for i in range(7, -1, -1):
        a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
        xp = P.paper_step(xp, lambda xc, g: eps(xc, i), wins, h, w, a_t, a_prev)
        xr = G.paper_step(xr, lambda xc, g, r: eps(xc, i) + r, masks, wins, h, w, a_t, a_prev)
        assert np.array_equal(xp, xr), i


def test_regions_helper_refuses_odd_sizes():
    from lib.model_zoo.regions import regions
    with pytest.raises(ValueError, match="multiples of 8"):
        regions(None, None, _cinfo(), _regions(), height=500, width=512)
