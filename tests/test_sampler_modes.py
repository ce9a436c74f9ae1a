"""The sampling modes together, CPU side: for every sampler, entry point and subset of the optional inputs, the refusal a call
raises (its type, a message substring and which one wins when two rules are broken) or that it gets past every check to the
sampler's 'no CPU path' error, and how many values it draws from torch's CPU generator on the way.  The model is a CPU fake, so
nothing here touches a device.  The draws on the way: the inpainting key (inpaint.py), then the SDE key of DPMSolverSDESampler at
eta > 0 (dpm_solver.py), after every mode is built; the bootstrapping key of regions.py is drawn at the walk's start, after the
device check, so no call here draws it."""
import itertools

import numpy as np
import pytest
import torch

from test_edit import _fake_model, _inversion

INPUTS = ("x0", "xt", "inpaint_mask", "inversion", "prompt_edit", "windows", "regions", "sag")
SUBSETS = [s for r in range(len(INPUTS) + 1) for s in itertools.combinations(INPUTS, r)]
NO_CPU = (RuntimeError, "no CPU path")


def expected(sampler, entry, given, text):
    """-> (exception type, message substring, 64-bit draws from the CPU generator) of one call."""
    if entry == "p_sample":
        if sampler in ("dpm", "sde0", "sde1"):
            return NotImplementedError, "no single-step form", 0
        for k, msg in (("prompt_edit", "a prompt edit spans the walk"), ("windows", "window fusion runs inside the sampler's walk"),
                       ("regions", "region prompts run inside the sampler's walk"),
                       ("sag", "self-attention guidance runs inside the sampler's walk")):
            if k in given:
                return NotImplementedError, msg, 0
        return NO_CPU + (0,)
    if sampler == "plms":
        for k, msg in (("inpaint_mask", "has no inpainting"), ("prompt_edit", "has no prompt editing"),
                       ("windows", "has no window fusion"), ("regions", "has no region prompts"),
                       ("inversion", "cannot sample from an inversion"), ("sag", "has no self-attention guidance")):
            if k in given:
                return NotImplementedError, "PLMSSampler " + msg, 0
        return NO_CPU + (0,)
    sde_key = int(sampler == "sde1")
    if "sag" in given:          # sag.py: SAG is the first mode built
        for k, msg in (("windows", "SAG with windows"), ("regions", "SAG with regions"), ("prompt_edit", "SAG with prompt_edit")):
            if k in given:
                return NotImplementedError, msg, 0
        if text:
            return ValueError, "SAG needs an image latent", 0
    if "regions" in given:      # regions.py: the windows given with regions are the region walk's layout
        if "prompt_edit" in given:
            return NotImplementedError, "regions with prompt_edit", 0
        if "inversion" in given:
            return NotImplementedError, "regions cannot sample from an inversion", 0
        if text:
            return ValueError, "regions need an image latent", 0
    elif "windows" in given:
        if "prompt_edit" in given:
            return NotImplementedError, "windows with prompt_edit", 0
        if "inversion" in given:
            return NotImplementedError, "windows cannot sample from an inversion", 0
        if text:
            return ValueError, "windows need an image latent", 0
    if "prompt_edit" in given:
        for k in ("x0", "inpaint_mask", "inversion"):
            if k in given:
                return ValueError, f"'prompt_edit' does not combine with '{k}'", 0
        if text:
            return ValueError, "a text latent cannot be edited", 0
    if "inversion" in given:
        for k in ("xt", "x0"):
            if k in given:
                return ValueError, f"x_info['{k}'] cannot be given with 'inversion'", 0
        if text:
            return ValueError, "differs from the inversion's", 0
        return NO_CPU + (sde_key,)  # an inpaint_mask blends against the trajectory: nothing is drawn for it
    if "inpaint_mask" in given:
        if text:
            return ValueError, "inpainting needs an image latent", 0
        if "x0" not in given:
            return ValueError, "inpaint_mask needs x_info['x0']", 0
        return NO_CPU + (1 + sde_key,)  # the Philox key
    return NO_CPU + (sde_key,)


def _inputs(given, text, entry="sample", bs=2):
    from lib.model_zoo.panorama import Windows
    from lib.model_zoo.prompt_edit import PromptEdit
    from lib.model_zoo.regions import Region, Regions
    from lib.model_zoo.sag import SelfAttentionGuidance
    shape = [bs, 768] if text else [bs, 4, 8, 8]
    x_info = {"type": "text" if text else "image", "x": torch.zeros(shape)}
    if "x0" in given:
        x_info.update(x0=torch.zeros(shape), x0_forward_timesteps=2)
    if "xt" in given:
        x_info["xt"] = torch.zeros(shape)
    if "inpaint_mask" in given:
        x_info["inpaint_mask"] = torch.ones(1, 1, 8, 8)
    if "inversion" in given:
        x_info["inversion"] = _inversion(bs=bs)
    if "windows" in given:
        x_info["windows"] = Windows(size=8, stride=4)
    if "regions" in given:
        c = torch.zeros(bs, 77, 768)
        x_info["regions"] = Regions([Region(torch.ones(1, 8, 8), [c, c] if entry == "sample_multicontext" else c)],
                                    bootstrap_steps=2, backgrounds=torch.zeros(3, 4))
    if "sag" in given:
        x_info["sag"] = SelfAttentionGuidance(0.75)
    c_infos = [{"type": "text", "conditioning": torch.zeros(bs, 77, 768), "unconditional_conditioning": torch.zeros(bs, 77, 768),
                "unconditional_guidance_scale": 7.5} for _ in range(2)]
    if "prompt_edit" in given:
        c_infos[0]["prompt_edit"] = PromptEdit(np.eye(77)[None], np.zeros((1, 77)))
    return shape, x_info, c_infos


def _call(S, entry, shape, x_info, c_infos, eta=None):
    kw = {} if eta is None else {"eta": eta}
    if entry == "sample":
        return S.sample(steps=5, shape=shape, x_info=x_info, c_info=c_infos[0], verbose=False, **kw)
    if entry == "sample_multicontext":
        return S.sample_multicontext(steps=5, shape=shape, x_info=x_info, c_info_list=c_infos, verbose=False, **kw)
    S.make_schedule(5, verbose=False)
    return S.p_sample_ddim(x_info, c_infos[0], torch.zeros(shape[0], dtype=torch.long), 4)


def _draws_after(n):
    """torch's CPU generator state after n 64-bit draws from seed 0"""
    torch.manual_seed(0)
    for _ in range(n):
        torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)
    return torch.get_rng_state()


@pytest.mark.parametrize("text", [False, True], ids=["image", "text"])
@pytest.mark.parametrize("entry", ["sample", "sample_multicontext", "p_sample"])
@pytest.mark.parametrize("sampler", ["ddim", "dpm", "plms", "sde0", "sde1"])
def test_combination_matrix(sampler, entry, text):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler, DPMSolverSDESampler
    from lib.model_zoo.plms import PLMSSampler
    cls = {"ddim": DDIMSampler, "dpm": DPMSolverSampler, "plms": PLMSSampler, "sde0": DPMSolverSDESampler,
           "sde1": DPMSolverSDESampler}[sampler]
    eta = {"sde0": 0.0, "sde1": 0.5}.get(sampler)
    states = [_draws_after(n) for n in range(3)]
    for given in SUBSETS:
        exc, match, draws = expected(sampler, entry, given, text)
        shape, x_info, c_infos = _inputs(given, text, entry)
        S = cls(_fake_model())
        torch.manual_seed(0)
        with pytest.raises(exc) as info:
            _call(S, entry, shape, x_info, c_infos, eta)
        assert match in str(info.value), (given, str(info.value))
        assert torch.equal(torch.get_rng_state(), states[draws]), (given, draws)


@pytest.mark.parametrize("steps", [67, 68, 69, 70])
def test_step_counted_arguments_on_the_short_karras_grid(steps):
    """From 67 steps on the Karras grid has fewer points than steps.  Every argument counted in steps counts the walk's grid
    points: a prompt edit's windows are fractions of the walk's length, bootstrap_steps and x0_forward_timesteps lie on it."""
    from lib.model_zoo.dpm_solver import DPMSolverSDESampler
    from lib.model_zoo.prompt_edit import PromptEdit
    from lib.model_zoo.regions import Region, Regions
    S = DPMSolverSDESampler(_fake_model(), grid="karras")
    S.make_schedule(steps, verbose=False)
    T = len(S.ddim_timesteps)
    assert T == steps - 1
    # the tables a prompt edit fills for a walk of T steps (the sampler passes T = the walk's length: test_mode_walks_gpu reads
    # them back from the device after a 68-step Karras walk)
    ed = PromptEdit(np.stack([np.eye(77)] * 2), np.zeros((2, 77)), cross_steps=0.8, self_steps=0.4)
    tabs = ed.tables(T, True)
    ident = np.arange(6)
    for name, frac in (("cross", 0.8), ("self", 0.4)):
        edited = [idx for idx in range(T) if not np.array_equal(tabs[name][idx, 0], ident)]
        assert edited == list(range(T - int(np.floor(frac * T)), T)), name      # walk positions 0 .. floor(frac T) - 1
    c = torch.zeros(2, 77, 768)
    cinfo = {"type": "text", "conditioning": c, "unconditional_conditioning": c, "unconditional_guidance_scale": 7.5}
    for boot, exc in ((T, RuntimeError), (T + 1, ValueError)):          # T + 1 == steps
        regs = Regions([Region(torch.ones(1, 8, 8), c)], bootstrap_steps=boot, backgrounds=torch.zeros(3, 4))
        with pytest.raises(exc) as info:
            S.sample(steps=steps, shape=[2, 4, 8, 8], x_info={"type": "image", "regions": regs}, c_info=cinfo, verbose=False)
        assert (f"[0, {T}]" if exc is ValueError else "no CPU path") in str(info.value), boot
    for k in (T, T + 3):
        with pytest.raises(ValueError, match=f"below the grid's {T} points, got {k}"):
            S._initial_latent([2, 4, 8, 8], {"x0": torch.zeros(2, 4, 8, 8), "x0_forward_timesteps": k}, torch.float32, "cpu")
