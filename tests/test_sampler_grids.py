"""The samplers' time grids (make_ddim_timesteps, the `grid` option): 'trailing' and 'karras' against their restatement from
diffusers / k-diffusion (oracle/dpm_sde_oracle.py), their shape, 'uniform' unchanged, the refusals, and the grid reaching every
sampler and DiffEdit's mask level."""
import types

import numpy as np
import pytest
import torch

from oracle import dpm_sde_oracle as G
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]


def _grid(name, n):
    from lib.model_zoo.diffusion_utils import make_ddim_timesteps
    return make_ddim_timesteps(name, n, 1000, verbose=False, alphas_cumprod=AC)


@pytest.mark.parametrize("name", ["trailing", "karras"])
def test_grid_matches_the_restatement_for_2_to_500_steps(name):
    for n in range(2, 501):
        got = _grid(name, n)
        want = G.trailing_grid(n) if name == "trailing" else G.karras_grid(AC.numpy(), n)
        assert np.array_equal(got, want), (name, n, got, want)


def test_grid_shapes():
    for n in range(2, 501):
        t, k = _grid("trailing", n), _grid("karras", n)
        for g in (t, k):
            assert np.all(np.diff(g) > 0) and g[-1] == 999, n
        assert len(t) == n and t[0] == int(np.round(1000 / n)) - 1, n
        assert k[0] == 1 and len(k) <= n, n
    assert list(_grid("trailing", 20)) == list(range(49, 1000, 50))
    assert list(_grid("trailing", 15)) == [66, 132, 199, 266, 332, 399, 466, 532, 599, 666, 732, 799, 866, 932, 999]
    k20 = list(_grid("karras", 20))
    assert len(k20) == 20 and k20[:6] == [1, 4, 11, 25, 51, 94] and k20[-3:] == [924, 963, 999]
    assert len(_grid("karras", 50)) == 50
    assert len(_grid("karras", 100)) == 98, "the low sigmas of 100 Karras points round onto 98 distinct timesteps"


def test_uniform_and_quad_are_unchanged():
    from lib.model_zoo.diffusion_utils import make_ddim_timesteps
    for n in (1, 5, 14, 20, 50, 333, 1000):
        assert np.array_equal(make_ddim_timesteps("uniform", n, 1000, verbose=False), O.make_ddim_timesteps(n))
        assert np.array_equal(make_ddim_timesteps("quad", n, 1000, verbose=False),
                              ((np.linspace(0, np.sqrt(800), n)) ** 2).astype(int) + 1)


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def test_refusals():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.diffusion_utils import make_ddim_timesteps
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler
    from lib.model_zoo.plms import PLMSSampler
    for cls in (DDIMSampler, PLMSSampler, DPMSolverSampler, DPMSolverSDESampler):
        for bad in ("Karras", "linspace", "quad", None, 3):
            with pytest.raises(ValueError, match="grid"):
                cls(_fake_model(), grid=bad)
    for n in (0, 1):
        with pytest.raises(ValueError, match="at least 2"):
            make_ddim_timesteps("karras", n, 1000, verbose=False, alphas_cumprod=AC)
        with pytest.raises(ValueError, match="at least 2"):
            DDIMSampler(_fake_model(), grid="karras").make_schedule(n, verbose=False)
    with pytest.raises(ValueError, match="alphas_cumprod"):
        make_ddim_timesteps("karras", 10, 1000, verbose=False)
    with pytest.raises(NotImplementedError):
        make_ddim_timesteps("cosine", 10, 1000, verbose=False)


@pytest.mark.parametrize("name", ["uniform", "trailing", "karras"])
def test_every_sampler_walks_its_grid(name):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler
    from lib.model_zoo.plms import PLMSSampler
    for cls in (DDIMSampler, PLMSSampler, DPMSolverSampler, DPMSolverSDESampler):
        S = cls(_fake_model(), grid=name) if name != "uniform" else cls(_fake_model())
        assert S.grid == name
        S.make_schedule(20, verbose=False)
        want = G.grid(name, 20, AC.numpy())
        assert np.array_equal(S.ddim_timesteps, want), cls
        assert np.array_equal(np.asarray(S.ddim_alphas), AC.numpy()[want]), cls
        # an explicit discretisation still wins over the sampler's grid
        S.make_schedule(20, ddim_discretize="uniform", verbose=False)
        assert np.array_equal(S.ddim_timesteps, O.make_ddim_timesteps(20)), cls


@pytest.mark.parametrize("name", ["uniform", "trailing", "karras"])
def test_diffedit_mask_follows_its_grid(name, monkeypatch):
    """diffedit_mask noises x0 to t_{k-1} of the grid it is given: captured at the timestep embedding, before any kernel runs."""
    from lib.model_zoo import edit
    seen = {}

    class Stop(Exception):
        pass

    def emb(t, *a, **k):
        seen["t"] = int(t[0])
        raise Stop

    ops = types.SimpleNamespace(nchw_to_nhwc=lambda x: x, axpby=lambda a, b, s, t: a, timestep_embedding=emb)
    monkeypatch.setattr(edit, "_ops", lambda: ops)
    net = types.SimpleNamespace(num_timesteps=1000, alphas_cumprod=AC, device="cpu", time_source=lambda *a: 0,
                                diffuser=[types.SimpleNamespace(model_channels=64)])
    c = {"type": "text", "conditioning": torch.zeros(1, 77, 768), "unconditional_conditioning": torch.zeros(1, 77, 768),
         "unconditional_guidance_scale": 1.0}
    steps, strength = 20, 0.5
    with pytest.raises(Stop):
        edit.diffedit_mask(net, torch.zeros(1, 4, 8, 8), c, c, steps=steps, strength=strength, n_draws=1, grid=name)
    assert seen["t"] == int(G.grid(name, steps, AC.numpy())[int(steps * strength) - 1])
