"""Panoramas, CPU side (lib/model_zoo/panorama.py): the window layout and its cover tables, every refusal of the samplers, and the
oracle (oracle/panorama_oracle.py): its paper-form DDIM average against the eps average on an analytic eps function in fp64, and a
one-window layout reducing its walk to the plain walk.  The C entry points a panorama runs are the region ones at R = 0, whose
argument checks tests/test_regions.py covers."""
import types

import numpy as np
import pytest
import torch

from oracle import dpm_solver_oracle as D
from oracle import panorama_oracle as P
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def _cover_sets(lay):
    """per element, the covering window indices in ascending order, read from the cover tables"""
    out = {}
    for y in range(lay.H):
        ys = range(*lay.cover_y[y])
        for x in range(lay.W):
            a0, a1, b0, b1 = lay.cover_x[x]
            xs = list(range(a0, a1)) + list(range(b0, b1))
            out[y, x] = [iy * lay.nx + ix for iy in ys for ix in xs]
    return out


CASES = [(64, 256, 64, 8, False), (64, 256, 64, 16, False), (64, 256, 64, 16, True), (16, 40, 16, 8, False),
         (32, 32, 16, 8, False), (16, 40, 16, 8, True), (24, 20, 16, 7, False), (8, 12, 64, 8, False), (40, 40, 16, 5, True),
         (64, 64, 64, 8, False), (16, 48, 16, 16, True)]


@pytest.mark.parametrize("H,W,size,stride,circular", CASES)
def test_layout(H, W, size, stride, circular):
    from lib.model_zoo.panorama import Windows, layout
    lay = layout(Windows(size, stride, circular), H, W)
    h, w, wins = P.windows(H, W, size, stride, circular)
    # sides clamp to the canvas; the origins are the oracle's, in the same window order
    assert (lay.h, lay.w) == (min(size, H), min(size, W)) == (h, w)
    assert [(int(oy), int(ox)) for oy in lay.oy for ox in lay.ox] == wins
    assert lay.nwin == len(wins) == lay.ny * lay.nx
    for o, L, side, wrap in ((lay.oy, H, lay.h, False), (lay.ox, W, lay.w, circular)):
        assert o[0] == 0 and np.all(np.diff(o) > 0)
        if wrap:
            assert list(o) == list(range(0, L, stride))
        else:
            assert o[-1] == L - side, "the last window is flush with the far edge"
            assert np.all(np.diff(o)[:-1] == stride) and 0 < np.diff(o)[-1] <= stride if len(o) > 1 else True
    # every element is covered, and the tables list exactly the covering windows in ascending order
    covers = _cover_sets(lay)
    counts = lay.counts()
    for (y, x), gs in covers.items():
        want = [g for g, (oy, ox) in enumerate(wins) if oy <= y < oy + h and (x - ox) % W < w]
        assert gs == want and len(gs) >= 1, (y, x)
        assert counts[y, x] == len(gs)
    if not circular:
        assert all((x - ox) % W == x - ox for (_, ox) in wins for x in range(ox, ox + w)), "no window wraps"


def test_layout_shapes_of_the_workload():
    """512x2048 (latent 64x256): 25 windows at stride 8, 13 at stride 16; a 360-degree layout at stride 16 has 16"""
    from lib.model_zoo.panorama import Windows, layout
    assert layout(Windows(64, 8), 64, 256).nwin == 25
    assert layout(Windows(64, 16), 64, 256).nwin == 13
    lay = layout(Windows(64, 16, circular=True), 64, 256)
    assert lay.nwin == 16 and np.all(lay.counts() == 4)
    assert layout(Windows(64, 8), 64, 64).nwin == 1, "a window equal to the canvas"
    lay = layout(Windows(64, 8), 40, 24)                # clamped to a small canvas: one window, the canvas itself
    assert (lay.h, lay.w, lay.nwin) == (40, 24, 1) and np.all(lay.counts() == 1)
    assert [c for c in layout(Windows(64, 8), 64, 256).chunks(8)] == [(0, 8), (8, 8), (16, 8), (24, 1)]
    assert layout(Windows(64, 16), 64, 256).chunks(13) == [(0, 13)]


def test_table_packs_cover_x_first():
    from lib.model_zoo.panorama import Windows, layout
    lay = layout(Windows(16, 8, True), 16, 40)
    tab, offs = lay.table()
    assert tab.dtype == np.int32 and offs["cover_x"][0] == 0, "cover_x rows are read as int4: they lead the table"
    for name in ("cover_x", "cover_y", "oy", "ox"):
        o, n = offs[name]
        assert np.array_equal(tab[o:o + n], getattr(lay, name).ravel())


def _cinfo(**kw):
    return dict({"type": "text", "conditioning": torch.zeros(1, 77, 768), "unconditional_conditioning": torch.zeros(1, 77, 768),
                 "unconditional_guidance_scale": 7.5}, **kw)


def _samplers():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return [DDIMSampler(_fake_model()), DPMSolverSampler(_fake_model())]


def test_windows_refusals():
    from lib.model_zoo.panorama import Windows
    for bad in (dict(size=7), dict(size=0), dict(size=64.0), dict(stride=0), dict(stride=65), dict(size=16, stride=17),
                dict(stride=-8), dict(stride=8.0)):
        with pytest.raises(ValueError, match="Windows"):
            Windows(**bad)
    Windows(size=8, stride=8)
    Windows(size=64, stride=1)


@pytest.mark.parametrize("multi", [False, True])
def test_sampler_refusals(multi):
    """Every refusal is raised before any device work (the fake model is on the CPU, where a call that passed them would raise
    RuntimeError instead)."""
    from lib.model_zoo.panorama import Windows
    bs, H, W = 1, 16, 40
    shape = [bs, 4, H, W]

    def run(S, shape, x_info, **ci):
        if multi:
            return S.sample_multicontext(steps=5, shape=shape, x_info=x_info, c_info_list=[_cinfo(**ci), _cinfo()], verbose=False)
        return S.sample(steps=5, shape=shape, x_info=x_info, c_info=_cinfo(**ci), verbose=False)

    for S in _samplers():
        with pytest.raises(ValueError, match="text latent"):
            run(S, [bs, 768], {"type": "text", "windows": Windows(16, 8)})
        with pytest.raises(ValueError, match="multiple of the stride"):
            run(S, shape, {"type": "image", "windows": Windows(16, 16, circular=True)})
        with pytest.raises(ValueError, match="panorama.Windows"):
            run(S, shape, {"type": "image", "windows": (64, 8)})
        with pytest.raises(NotImplementedError, match="prompt_edit"):
            run(S, shape, {"type": "image", "windows": Windows(16, 8)}, prompt_edit=object())
        with pytest.raises(NotImplementedError, match="inversion"):
            run(S, shape, {"type": "image", "windows": Windows(16, 8), "inversion": object()})
        # valid inputs pass the checks and reach the device check: plain, circular, img2img start, inpainting
        for x_info in ({"type": "image", "windows": Windows(16, 8)}, {"type": "image", "windows": Windows(16, 8, circular=True)},
                       {"type": "image", "windows": Windows(16, 4), "x0": torch.zeros(1, 4, H, W), "x0_forward_timesteps": 3},
                       {"type": "image", "windows": Windows(16, 8), "x0": torch.zeros(1, 4, H, W),
                        "inpaint_mask": torch.ones(1, 1, H, W)}):
            with pytest.raises(RuntimeError, match="no CPU path"):
                run(S, shape, x_info)


def test_plms_and_the_single_step_api_refuse_windows():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.panorama import Windows
    from lib.model_zoo.plms import PLMSSampler
    S = PLMSSampler(_fake_model())
    with pytest.raises(NotImplementedError, match="window fusion"):
        S.sample(steps=5, shape=[1, 4, 16, 40], x_info={"type": "image", "windows": Windows(16, 8)}, c_info=_cinfo(),
                 verbose=False)
    S = DDIMSampler(_fake_model())
    S.make_schedule(5, verbose=False)
    with pytest.raises(NotImplementedError, match="window fusion"):
        S.p_sample_ddim({"type": "image", "x": torch.zeros(1, 4, 16, 40), "windows": Windows(16, 8)}, _cinfo(),
                        torch.zeros(1, dtype=torch.long), 0)


def test_panorama_helper_refuses_odd_sizes():
    from lib.model_zoo.panorama import panorama
    with pytest.raises(ValueError, match="multiples of 8"):
        panorama(None, None, _cinfo(), height=500, width=2048)


# ---- the oracle on an analytic eps function ---------------------------------------------------------------------------------------
def _eps(i):
    """an eps that depends on the crop, the window and the step, so overlapping windows disagree"""
    return lambda xc, g: np.tanh(0.7 * xc) * (1.0 + 0.1 * g) + 0.03 * (g - 2) + 0.01 * i


@pytest.mark.parametrize("H,W,size,stride,circular", [(16, 40, 16, 8, False), (32, 32, 16, 8, False), (16, 40, 16, 8, True),
                                                      (24, 20, 16, 7, False)])
def test_oracle_paper_form_equals_the_eps_average(H, W, size, stride, circular):
    """DDIM is x' = a x + b eps per element with the same a, b in every window, so the average of the windows' x' is the update of
    the average eps: the product's form equals the paper's, in fp64 up to rounding."""
    ts = O.make_ddim_timesteps(10)
    sched = O.ddim_schedule(AC, 10)
    g = np.random.default_rng(H * W + stride)
    x = g.standard_normal((2, 4, H, W))
    h, w, wins = P.windows(H, W, size, stride, circular)
    assert len(wins) > 1
    for i in (9, 4, 0):
        a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
        paper = P.paper_step(x, _eps(i), wins, h, w, a_t, a_prev)
        via_eps = P.ddim_update(x, P.eps_average(x, _eps(i), wins, h, w), a_t, a_prev)
        assert np.abs(paper - via_eps).max() <= 1e-13 * np.abs(paper).max(), i
        # the windows disagree, so the average is not any single window's step
        one = P.ddim_update(x, P.eps_average(x, lambda xc, gg: _eps(i)(xc, 0), wins, h, w), a_t, a_prev)
        assert np.abs(paper - one).max() > 1e-3
        x = paper
    assert ts.shape[0] == 10


def test_oracle_one_window_is_the_plain_walk():
    """A window equal to the canvas: the eps average is the window's eps exactly, so the windowed walks are the plain ones bit for
    bit (DPM-Solver++ through dpm_solver_oracle.walk, DDIM through the paper-form step)."""
    H, W = 16, 24
    h, w, wins = P.windows(H, W, 64, 8)
    assert (h, w, wins) == (H, W, [(0, 0)])
    ts = O.make_ddim_timesteps(8)
    x = np.random.default_rng(1).standard_normal((1, 4, H, W))
    eps = lambda xv, i: np.tanh(0.7 * xv) + 0.01 * i
    for order in (1, 2, 3):
        plain = D.walk(x, eps, AC.numpy(), ts, order)
        windowed = D.walk(x, lambda xv, i: P.eps_average(xv, lambda xc, g: eps(xc, i), wins, h, w), AC.numpy(), ts, order)
        assert np.array_equal(plain, windowed), order
    sched = O.ddim_schedule(AC, 8)
    xp, xw = x, x
    for i in range(7, -1, -1):
        a_t, a_prev = float(sched["alphas"][i]), float(sched["alphas_prev"][i])
        xp = P.ddim_update(xp, eps(xp, i), a_t, a_prev)
        xw = P.paper_step(xw, lambda xc, g: eps(xc, i), wins, h, w, a_t, a_prev)
        assert np.array_equal(xp, xw), i
