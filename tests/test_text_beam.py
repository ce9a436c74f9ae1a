"""Text decoder beam search, CPU side: the fp64 oracle against exhaustive search, greedy decoding, the tie rule and the forced
<EOS>; the C ABI's argument checks of the beam entry points; decode()'s checks of num_beams."""
import math

import numpy as np
import pytest
import torch

from oracle.text_beam_oracle import BeamState, beam_search, beam_step, log_softmax64, scored_tokens

BOS, EOS = 0, 2


def toy_logits(V, seed, dup=False):
    """logits_fn of beam_search: fp32 logits of each row's next token, a fixed function of its history."""
    def fn(s, hist):
        out = np.empty((hist.shape[0], V), dtype=np.float32)
        for r, h in enumerate(hist):
            rng = np.random.default_rng([seed] + [int(t) for t in h])
            out[r] = (rng.standard_normal(V) * 2).astype(np.float32)
            if dup:
                out[r, V - 1] = out[r].max()              # an exact tie for the maximum
        return out
    return fn


def exhaustive(fn, V, max_len, temperature):
    """every hypothesis (chosen tokens until a chosen <EOS>, or <EOS> forced after token max_len - 2) with its fp64 score"""
    out = {}

    def walk(ids, score):
        s = len(ids) - 1
        lp = log_softmax64(fn(s, np.array([ids])), temperature)[0]
        for v in range(V):
            nxt, sc = ids + [v], score + lp[v]
            if v == EOS:
                out[tuple(nxt)] = sc
            elif s + 1 >= max_len - 2:
                out[tuple(nxt + [EOS])] = sc
            else:
                walk(nxt, sc)
    walk([BOS], 0.0)
    return out


@pytest.mark.parametrize("temperature", [1.0, 0.7])
def test_oracle_wide_beam_equals_exhaustive_search(temperature):
    V, max_len = 3, 6                                     # at most 4 chosen tokens: 3^4 = 81 hypotheses at most
    fn = toy_logits(V, 11)
    want = exhaustive(fn, V, max_len, temperature)
    K = V ** (max_len - 2)
    ranked, _ = beam_search(fn, 1, K, BOS, EOS, max_len, temperature, length_penalty=0.0)
    got = {tuple(int(t) for t in ids): sc for ids, sc, _ in ranked[0] if math.isfinite(sc)}
    assert got.keys() == want.keys()
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12 * abs(want[k]), k
    best = max(want, key=want.get)
    assert tuple(int(t) for t in ranked[0][0][0]) == best
    # length_penalty 1 ranks by the mean over scored tokens
    ranked1, _ = beam_search(fn, 1, K, BOS, EOS, max_len, temperature, length_penalty=1.0)
    norm = {k: v / scored_tokens(len(k), max_len) for k, v in want.items()}
    assert tuple(int(t) for t in ranked1[0][0][0]) == max(norm, key=norm.get)


@pytest.mark.parametrize("dup", [False, True])
def test_oracle_width_one_is_stepwise_argmax(dup):
    V, max_len = 40, 12
    fn = toy_logits(V, 5, dup=dup)
    ranked, _ = beam_search(fn, 1, 1, BOS, EOS, max_len)
    ids = [BOS]
    while True:
        s = len(ids) - 1
        v = int(np.argmax(fn(s, np.array([ids]))[0]))      # the first of equal maxima: the lowest token id
        ids.append(v)
        if v == EOS:
            break
        if s + 1 >= max_len - 2:
            ids.append(EOS)
            break
    assert [int(t) for t in ranked[0][0][0]] == ids


def test_oracle_tie_rule():
    """equal scores go to the lower parent beam, then the lower token id"""
    K, V = 3, 8
    st = BeamState.start(1, K, BOS, EOS)
    st.scores[:] = -1.0
    row = np.full(V, -3.0, dtype=np.float32)
    row[[5, 3]] = 1.0
    logits = np.stack([row] * K)
    new, trace, margins = beam_step(st, logits, K, 2, EOS, 30)
    assert [tuple(int(x) for x in t[:2]) for t in trace] == [(0, 3), (0, 5), (1, 3)]
    assert trace[0, 2] == trace[2, 2] and margins[0] == math.inf
    assert list(new.src[:, 2]) == [0, 0, 1]
    # a finished beam is one candidate, itself; it outranks an equal-scoring later parent's children
    st.done[0] = True
    st.scores[0] = -1.0 + float(log_softmax64(logits, 1.0)[0, 3])
    new, trace, _ = beam_step(st, logits, K, 2, EOS, 30)
    assert [tuple(int(x) for x in t[:2]) for t in trace] == [(0, -1), (1, 3), (1, 5)]
    assert new.done.tolist() == [True, False, False]


def test_oracle_forced_eos_is_not_scored():
    V, max_len = 6, 4                                      # steps 0 and 1; token 2 (s + 1 == max_len - 2) gets <EOS> appended
    fn = toy_logits(V, 3)
    fn2 = lambda s, h: np.where(np.arange(V) == EOS, np.float32(-1e30), fn(s, h)).astype(np.float32)   # <EOS> never chosen
    ranked, st = beam_search(fn2, 1, 1, BOS, EOS, max_len)
    ids, score, norm = ranked[0][0]
    assert len(ids) == 4 and ids[-1] == EOS and st.lengths[0] == 4
    lp = [log_softmax64(fn2(s, ids[None, :s + 1]), 1.0)[0, ids[s + 1]] for s in range(2)]
    assert score == lp[0] + lp[1] and norm == score / 2


def test_beam_step_and_attention_src_check_arguments_before_launch():
    """bad arguments return VDB_ERR_INVALID with a message (the fake addresses are never touched)."""
    from vdb200._lib import lib
    x, out, step = 0x10000, 0x30000, 0x40000

    def beam(R=4, V=50260, temp=1.0, K=2, logits=x, tokens=out, src=out, scores=out):
        return lib.vdb_textdec_beam_step(logits, R, V, V, temp, K, tokens, 33, src, 32, scores, out, out, step, 50259, 30,
                                         out, out, None, None, None)
    for kw, msg in ((dict(R=17, K=1), b"R = n * K <= 16"), (dict(R=18, K=2), b"R = n * K <= 16"), (dict(R=6, K=4), b"R = n * K"),
                    (dict(K=0), b"1 <= K <= 16"), (dict(K=17, R=17), b"1 <= K <= 16"), (dict(logits=None), b"null"),
                    (dict(tokens=None), b"null"), (dict(src=None), b"null"), (dict(scores=None), b"null"),
                    (dict(V=53249), b"53248"), (dict(V=1, K=2), b"K <= V"), (dict(temp=0.0), b"temperature"),
                    (dict(temp=-1.0), b"temperature"), (dict(scores=out + 4), b"8-byte aligned"),
                    (dict(tokens=out + 2), b"4-byte aligned"), (dict(src=out + 1), b"4-byte aligned"),
                    (dict(logits=x + 2), b"4-byte aligned")):
        assert beam(**kw) == 1 and msg in lib.vdb_last_error(), (kw, lib.vdb_last_error())
    att = lambda R=4, src=out, qkv=x: lib.vdb_textdec_attention(qkv, 2304, x, 768, out, out, src, R, 12, 32, step, 0.125, out, 768,
                                                                None)
    assert att(R=17) == 1 and b"R <= 16" in lib.vdb_last_error()
    assert att(qkv=None) == 1 and b"null" in lib.vdb_last_error()
    assert att(src=out + 2) == 1 and b"aligned" in lib.vdb_last_error()
    # src = NULL is the plain path: it passes the null-pointer check, so the row count is what is refused
    assert att(src=None, R=17) == 1 and b"R <= 16" in lib.vdb_last_error()


def test_decode_rejects_bad_beam_arguments():
    from lib.model_zoo.optimus import optimus_vae_next
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=2)))
    z = torch.zeros(2, 768)
    for kw in (dict(num_beams=2, top_k=5), dict(num_beams=1, top_p=0.9), dict(num_beams=2.0), dict(num_beams=True),
               dict(num_beams=17), dict(num_beams=-1), dict(num_beams="4"), dict(num_beams=2, length_penalty=math.nan)):
        with pytest.raises(ValueError):
            m.decode(z, **kw)
        with pytest.raises(ValueError):
            m.decode_ids(z, **kw)
    with pytest.raises(ValueError):
        m.decode_ids(z, num_beams=2, return_logits=True)
    for K in (0, 17, 2.5):
        with pytest.raises(ValueError):
            m.decode_beams(z, K)
