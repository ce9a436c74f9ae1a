"""The option checks of the text decoder's entry points (decode, decode_ids, decode_beams, teacher_forced_logits), CPU side.

For every single bad option and every pair of bad options, across features (the top-k / nucleus cuts, beam search, the repetition
processors), the call raises the exception and message of the first check in the fixed order below, before any device work and
without drawing from torch's CPU generator.  A call whose options are all valid reaches require_cuda's RuntimeError (the latents
are on the CPU), again without a draw: the sampling seed is taken only after every check has passed."""
import itertools
import math

import pytest
import torch

MAX_BEAMS, MAX_LENGTH = 16, 30

# one bad value per row; the cases take every value alone and the first value of each option in pairs
BAD = {
    "repetition_penalty": (0.0, math.nan, 1e39, True),
    "no_repeat_ngram_size": (-1, 31, 2.0, None),
    "num_beams": (-1, 17, 2.0, True, "4"),
    "length_penalty": (math.nan, math.inf, "1.0", True),
    "top_k": (-1, 1.5, True, "40"),
    "top_p": (math.nan, -0.1, 1.01, None),
}
# the order in which the checks run: the first bad option in it is the one reported
FIRST = ("repetition_penalty", "no_repeat_ngram_size", "num_beams", "length_penalty")
MESSAGE = {
    "repetition_penalty": "optimus_vae_next: repetition_penalty must be a finite float > 0 (1: off), got {!r}",
    "no_repeat_ngram_size": f"optimus_vae_next: no_repeat_ngram_size must be an int in [0, {MAX_LENGTH}] (0: off), got {{!r}}",
    "num_beams": f"optimus_vae_next: num_beams must be an int in [0, {MAX_BEAMS}] (0: sampling), got {{!r}}",
    "length_penalty": "optimus_vae_next: length_penalty must be a finite float, got {!r}",
    "top_k": "optimus_vae_next: top_k must be an int >= 0 (0: no top-k cut), got {!r}",
    "top_p": "optimus_vae_next: top_p must be a finite float in [0, 1] (0 or 1: no nucleus cut), got {!r}",
}
BEAM_CUT = "optimus_vae_next: beam search (num_beams >= 1) takes no top_k / top_p cut"
BEAM_DRAW = "optimus_vae_next: beam search takes no uniforms and returns no logits"
NO_CUDA = "optimus_vae_next.decode: the H100 build has no CPU path"


@pytest.fixture(scope="module")
def m():
    from lib.model_zoo.optimus import optimus_vae_next
    return optimus_vae_next(decoder=dict(config=dict(n_layer=2)))


def _z():
    return torch.zeros(2, 768)


def _uniforms():
    return torch.zeros(2, 28, dtype=torch.float64)


def _sampling_cases():
    """(kwargs of decode_ids / decode, names of the bad options among them)"""
    cases = [({name: v}, {name}) for name, vals in BAD.items() for v in vals]
    cases += [({a: BAD[a][0], b: BAD[b][0]}, {a, b}) for a, b in itertools.combinations(BAD, 2)]
    # valid beam search with a sampling-only option; with that and a bad option of every feature
    beam_only = (dict(top_k=-1), dict(top_k=5), dict(top_p=0.9), dict(top_p=math.nan), dict(uniforms=True), dict(return_logits=True),
                 dict(top_k=5, uniforms=True), dict(top_p=0.5, return_logits=True))
    for kw in beam_only:
        cases.append(({"num_beams": 2, **kw}, set()))
        for name in FIRST:
            if name != "num_beams":
                cases.append(({"num_beams": 2, **kw, name: BAD[name][0]}, {name}))
    # sampling-only options with num_beams 0 are the sampler's, and cuts of valid values with bad options elsewhere
    cases += [(dict(num_beams=0, uniforms=True, top_k=-1), {"top_k"}), (dict(num_beams=0, return_logits=True), set()),
              (dict(num_beams=1, top_k=0, top_p=0.0), set()), (dict(top_k=40, top_p=0.9, repetition_penalty=1.2), set()),
              (dict(top_k=40, top_p=0.9, no_repeat_ngram_size=31), {"no_repeat_ngram_size"}),
              (dict(num_beams=4, length_penalty=0.0, repetition_penalty=1.3, no_repeat_ngram_size=2), set())]
    return cases


def _sampling_want(kw, bad):
    for name in FIRST:
        if name in bad:
            return ValueError, MESSAGE[name].format(kw[name])
    if kw.get("num_beams", 0):
        if "top_k" in kw and kw["top_k"] != 0 or "top_p" in kw and kw["top_p"] != 0.0:
            return ValueError, BEAM_CUT
        if kw.get("uniforms") or kw.get("return_logits"):
            return ValueError, BEAM_DRAW
        return RuntimeError, NO_CUDA
    for name in ("top_k", "top_p"):
        if name in bad:
            return ValueError, MESSAGE[name].format(kw[name])
    return RuntimeError, NO_CUDA


def _beam_cases():
    """(num_beams, kwargs of decode_beams, names of the bad options)"""
    rows = [(K, {}, {"num_beams"}) for K in BAD["num_beams"]] + [(0, {}, {"num_beams"}), (1, {}, set()), (16, {}, set())]
    rows += [(2, {name: v}, {name}) for name in FIRST if name != "num_beams" for v in BAD[name]]
    for a, b in itertools.combinations(FIRST, 2):
        kw = {n: BAD[n][0] for n in (a, b) if n != "num_beams"}
        rows.append((BAD["num_beams"][0] if "num_beams" in (a, b) else 2, kw, {a, b}))
        if "num_beams" in (a, b):
            rows.append((0, kw, {a, b}))
    return rows


def _beam_want(K, kw, bad):
    for name in FIRST:
        if name in bad:
            if name == "num_beams" and K == 0:
                continue                                   # 0 is in range: refused only after length_penalty is checked
            return ValueError, MESSAGE[name].format(K if name == "num_beams" else kw[name])
    if K == 0:
        return ValueError, "optimus_vae_next.decode_beams: num_beams must be >= 1, got 0"
    return RuntimeError, NO_CUDA


def _check(call, want):
    exc, msg = want
    torch.manual_seed(0)
    state = torch.get_rng_state()
    with pytest.raises(Exception) as info:
        call()
    assert type(info.value) is exc, (type(info.value), str(info.value), want)
    if exc is RuntimeError:
        assert str(info.value).startswith(msg), str(info.value)
    else:
        assert str(info.value) == msg
    assert torch.equal(torch.get_rng_state(), state), "the CPU generator was drawn from"


def _kwargs(kw):
    return {k: (_uniforms() if k == "uniforms" and v is True else v) for k, v in kw.items()}


@pytest.mark.parametrize("kw,bad", _sampling_cases(), ids=lambda v: repr(v) if isinstance(v, dict) else "")
def test_decode_ids_refusals(m, kw, bad):
    _check(lambda: m.decode_ids(_z(), **_kwargs(kw)), _sampling_want(kw, bad))


@pytest.mark.parametrize("kw,bad", [c for c in _sampling_cases() if not {"uniforms", "return_logits"} & set(c[0])],
                         ids=lambda v: repr(v) if isinstance(v, dict) else "")
def test_decode_refusals(m, kw, bad):
    _check(lambda: m.decode(_z(), **kw), _sampling_want(kw, bad))


@pytest.mark.parametrize("K,kw,bad", _beam_cases(), ids=lambda v: repr(v) if isinstance(v, (dict, int, float, str)) else "")
def test_decode_beams_refusals(m, K, kw, bad):
    _check(lambda: m.decode_beams(_z(), K, **kw), _beam_want(K, kw, bad))


@pytest.mark.parametrize("graph", [False, True])
def test_teacher_forced_logits_reaches_the_device_check(m, graph):
    ids = torch.full((2, 5), 50259, dtype=torch.long)
    _check(lambda: m.teacher_forced_logits(_z(), ids, graph=graph), (RuntimeError, NO_CUDA))
