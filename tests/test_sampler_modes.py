"""The sampling modes together, CPU side: for every sampler, entry point and subset of the optional inputs, the refusal a call
raises (its type, a message substring and which one wins when two rules are broken) or that it gets past every check to the
sampler's 'no CPU path' error, and how many values it draws from torch's CPU generator on the way.  The model is a CPU fake, so
nothing here touches a device."""
import itertools

import numpy as np
import pytest
import torch

from test_edit import _fake_model, _inversion

INPUTS = ("x0", "xt", "inpaint_mask", "inversion", "prompt_edit", "windows")
SUBSETS = [s for r in range(len(INPUTS) + 1) for s in itertools.combinations(INPUTS, r)]
NO_CPU = (RuntimeError, "no CPU path")


def expected(sampler, entry, given, text):
    """-> (exception type, message substring, 64-bit draws from the CPU generator) of one call."""
    if entry == "p_sample":
        if sampler == "dpm":
            return NotImplementedError, "no single-step form", 0
        if "prompt_edit" in given:
            return NotImplementedError, "a prompt edit spans the walk", 0
        if "windows" in given:
            return NotImplementedError, "window fusion runs inside the sampler's walk", 0
        return NO_CPU + (0,)
    if sampler == "plms":
        for k, msg in (("inpaint_mask", "has no inpainting"), ("prompt_edit", "has no prompt editing"),
                       ("windows", "has no window fusion"), ("inversion", "cannot sample from an inversion")):
            if k in given:
                return NotImplementedError, "PLMSSampler " + msg, 0
        return NO_CPU + (0,)
    if "windows" in given:
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
        return NO_CPU + (0,)        # an inpaint_mask blends against the trajectory: nothing is drawn
    if "inpaint_mask" in given:
        if text:
            return ValueError, "inpainting needs an image latent", 0
        if "x0" not in given:
            return ValueError, "inpaint_mask needs x_info['x0']", 0
        return NO_CPU + (1,)        # the Philox key
    return NO_CPU + (0,)


def _inputs(given, text, bs=2):
    from lib.model_zoo.panorama import Windows
    from lib.model_zoo.prompt_edit import PromptEdit
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
    c_infos = [{"type": "text", "conditioning": torch.zeros(bs, 77, 768), "unconditional_conditioning": torch.zeros(bs, 77, 768),
                "unconditional_guidance_scale": 7.5} for _ in range(2)]
    if "prompt_edit" in given:
        c_infos[0]["prompt_edit"] = PromptEdit(np.eye(77)[None], np.zeros((1, 77)))
    return shape, x_info, c_infos


def _call(S, entry, shape, x_info, c_infos):
    if entry == "sample":
        return S.sample(steps=5, shape=shape, x_info=x_info, c_info=c_infos[0], verbose=False)
    if entry == "sample_multicontext":
        return S.sample_multicontext(steps=5, shape=shape, x_info=x_info, c_info_list=c_infos, verbose=False)
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
@pytest.mark.parametrize("sampler", ["ddim", "dpm", "plms"])
def test_combination_matrix(sampler, entry, text):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    from lib.model_zoo.plms import PLMSSampler
    cls = {"ddim": DDIMSampler, "dpm": DPMSolverSampler, "plms": PLMSSampler}[sampler]
    states = [_draws_after(n) for n in range(3)]
    for given in SUBSETS:
        exc, match, draws = expected(sampler, entry, given, text)
        shape, x_info, c_infos = _inputs(given, text)
        S = cls(_fake_model())
        torch.manual_seed(0)
        with pytest.raises(exc) as info:
            _call(S, entry, shape, x_info, c_infos)
        assert match in str(info.value), (given, str(info.value))
        assert torch.equal(torch.get_rng_state(), states[draws]), (given, draws)
