"""Repetition penalty and no-repeat n-gram bans of the text decoder, CPU side: the numpy oracle (oracle/text_repetition_oracle.py)
against what Hugging Face's RepetitionPenaltyLogitsProcessor and NoRepeatNGramLogitsProcessor produced
(tests/golden/text_repetition.npz), the oracle's identities, the argument checks of vdb_textdec_repetition, and the checks of
decode / decode_ids / decode_beams, which must reject bad knobs before any device work."""
import math
import os

import numpy as np
import pytest
import torch

from oracle.text_repetition_oracle import banned_tokens, has_repeated_ngram, process

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def test_oracle_equals_the_hf_processors_bitwise():
    gold = dict(np.load(os.path.join(GOLD, "text_repetition.npz")))
    logits, tokens = gold["logits"], gold["tokens"]
    assert logits.dtype == np.float32 and len(gold["out"]) == len(gold["penalty"])
    hit = set()
    for i, (p, n, s) in enumerate(zip(gold["penalty"], gold["ngram"], gold["step"])):
        got = process(logits, tokens, int(s), None, float(p), int(n))
        assert np.array_equal(got.view(np.uint32), gold["out"][i].view(np.uint32)), (p, n, s)
        bans = np.isneginf(gold["out"][i]) & ~np.isneginf(process(logits, tokens, int(s), None, float(p), 0))
        if bans.any():
            hit.add((int(n), "below" if s < n - 1 else "at" if s == n - 1 else "above"))
    # HF banned tokens for every n of the fixture, at s = n - 1 and above; below, nothing (the spec's own rule)
    assert {h[0] for h in hit} == {1, 2, 3, 4, 30} and {h[1] for h in hit} == {"at", "above"}, sorted(hit)


def _case(R=3, V=40, seed=0):
    rng = np.random.default_rng(seed)
    logits = (rng.standard_normal((R, V)) * 3).astype(np.float32)
    logits[:, 0], logits[:, 1] = 0.0, -0.0
    tokens = rng.integers(0, 6, (R, 33))
    return logits, tokens


def test_identities():
    logits, tokens = _case()
    for s in (0, 5, 31):
        assert np.array_equal(process(logits, tokens, s, None, 1.0, 0).view(np.uint32), logits.view(np.uint32))
        out = process(logits, tokens, s, None, 1.0, 1)                      # n = 1 bans exactly the history
        for r in range(3):
            assert set(np.flatnonzero(np.isneginf(out[r]))) == set(tokens[r, :s + 1].tolist())
            keep = np.ones(40, bool)
            keep[tokens[r, :s + 1]] = False
            assert np.array_equal(out[r, keep], logits[r, keep])
    row = np.array([[2.0, -2.0, 8.0, 0.5]], np.float32)
    out = process(row, np.array([[0, 1, 0, 0, 1, 2]]), 5, None, 2.0, 0)     # ids 0 and 1 occur 3 and 2 times: penalised once
    assert out.tolist() == [[1.0, -4.0, 4.0, 0.5]]
    assert process(row, np.array([[0]]), 0, [1], 2.0, 1).tolist() == row.tolist()       # a finished row is left as it is


def test_ngram_rule():
    h = [5, 7, 5, 7, 5]
    assert banned_tokens(h, 2) == [7, 7] and banned_tokens(h, 3) == [7] and banned_tokens(h, 4) == [7]
    assert banned_tokens(h, 5) == [] and banned_tokens(h, 6) == [] and banned_tokens(h, 1) == h
    assert banned_tokens([3, 3, 3], 2) == [3, 3] and banned_tokens([1, 2], 3) == []
    assert has_repeated_ngram([1, 2, 1, 2], 2) and not has_repeated_ngram([1, 2, 3, 1, 3], 2)
    assert has_repeated_ngram([4, 4, 4], 2) and not has_repeated_ngram([4, 4], 2)


def test_ids_outside_the_vocabulary_are_ignored():
    logits, _ = _case(R=1, V=10)
    h = np.array([[-1, 10, 3, 10, 57, 3, -1, 10]])
    out = process(logits, h, 7, None, 2.0, 0)
    want = logits.copy()
    want[0, 3] = want[0, 3] * np.float32(2.0) if want[0, 3] < 0 else want[0, 3] / np.float32(2.0)
    assert np.array_equal(out, want)
    out = process(logits, h, 7, None, 1.0, 2)                                # -1 10 repeats: its continuation 3 is banned
    assert np.flatnonzero(np.isneginf(out[0])).tolist() == [3]
    assert np.isfinite(process(logits, h, 7, None, 1.0, 1)[0, [0, 1, 2, 4, 5, 6, 7, 8, 9]]).all()


def test_symbol_is_exported():
    from vdb200 import _lib
    assert hasattr(_lib.lib, "vdb_textdec_repetition") and "vdb_textdec_repetition" in _lib.SIGNATURES


def test_repetition_entry_point_checks_arguments_before_launch():
    """Every call here is refused before a launch (the fake addresses are never touched); both knobs off launch nothing."""
    from vdb200._lib import lib
    x, tok, done, step = 0x10000, 0x20000, 0x30000, 0x40000

    def rep(R=4, V=50260, ldl=50260, ldt=33, penalty=1.2, ngram=3, logits=x, tokens=tok, d=done, st=step):
        return lib.vdb_textdec_repetition(logits, R, V, ldl, tokens, ldt, d, st, penalty, ngram, None)
    before = lib.vdb_launch_count()
    for kw, msg in ((dict(R=0), b"R <= 16"), (dict(R=17), b"R <= 16"), (dict(V=0), b"V >= 1"), (dict(ldl=50259), b"ldl >= V"),
                    (dict(ldt=0), b"ldt >= 1"), (dict(penalty=0.0), b"penalty"), (dict(penalty=-1.2), b"penalty"),
                    (dict(penalty=math.nan), b"penalty"), (dict(penalty=math.inf), b"penalty"), (dict(ngram=-1), b"ngram"),
                    (dict(ngram=34), b"ngram"), (dict(logits=None), b"null"), (dict(tokens=None), b"null"), (dict(d=None), b"null"),
                    (dict(st=None), b"null"), (dict(logits=x + 2), b"4-byte aligned"), (dict(tokens=tok + 1), b"4-byte aligned"),
                    (dict(d=done + 2), b"4-byte aligned"), (dict(st=step + 3), b"4-byte aligned")):
        assert rep(**kw) == 1 and msg in lib.vdb_last_error(), (kw, lib.vdb_last_error())
    assert rep(penalty=1.0, ngram=0) == 0
    assert lib.vdb_launch_count() == before


BAD = (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=math.nan),
       dict(repetition_penalty=math.inf), dict(repetition_penalty=1e39), dict(repetition_penalty=1e-50),
       dict(repetition_penalty=True), dict(repetition_penalty="1.2"), dict(repetition_penalty=None),
       dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=31), dict(no_repeat_ngram_size=2.0),
       dict(no_repeat_ngram_size=True), dict(no_repeat_ngram_size="3"), dict(no_repeat_ngram_size=None))


def test_decode_rejects_bad_knobs_before_device_work():
    from lib.model_zoo.optimus import optimus_vae_next
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=2)))
    z = torch.zeros(2, 768)                                    # on the CPU: a check after the first launch would fail otherwise
    for kw in BAD:
        what = "repetition_penalty" if "repetition_penalty" in kw else "no_repeat_ngram_size"
        with pytest.raises(ValueError, match=what):
            m.decode_ids(z, **kw)
        with pytest.raises(ValueError, match=what):
            m.decode_ids(z, num_beams=2, **kw)
        with pytest.raises(ValueError, match=what):
            m.decode_beams(z, 2, **kw)
        with pytest.raises(ValueError, match=what):
            m.decode(z, **kw)
