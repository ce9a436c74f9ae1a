"""Prompt-to-Prompt, CPU side (lib/model_zoo/prompt_edit.py): the builders on a toy tokenizer (word positions, the replacement
mapper, the alignment, the equalizer), the window and flag tables, the fp64 identity between the factored form and P2P's edit
on the probabilities, every refusal (all raised before any device work), and the new C entry points' argument checks."""
import types

import numpy as np
import pytest
import torch

from oracle import vd_oracle as O

L = 77


class ToyTokenizer(object):
    """Words split into pieces of at most 4 characters; start 0, end 1, every piece its own id."""

    def __init__(self):
        self.vocab, self.inv = {}, {0: "<s>", 1: "</s>"}

    def _id(self, piece):
        if piece not in self.vocab:
            self.vocab[piece] = len(self.vocab) + 2
            self.inv[self.vocab[piece]] = piece
        return self.vocab[piece]

    def encode(self, text):
        ids = [0]
        for w in text.split(' '):
            ids += [self._id(w[i:i + 4]) for i in range(0, len(w), 4)]
        return ids + [1]

    def decode(self, ids):
        return "".join(self.inv[i] for i in ids)


def _pe():
    from lib.model_zoo import prompt_edit as pe
    return pe


def test_docstring_states_the_semantics():
    doc = " ".join(_pe().__doc__.split())
    for phrase in ("idx = T-1-i", "softmax(s q_src K(ctx_src)^T) V(ctx'_b)", "(attn_src M) * c", "3x3 max-pool (stride 1, pad 1)",
                   "floor(y h / H)", "false when the max is 0", "match +1, mismatch -1, gap -1", "prefers the diagonal, then a target insertion",
                   "threshold = 0.3, blend_start = 0, cross_steps = 0.8, self_steps = 0.4", "nothing changes",
                   "records them after its in-place edit"):
        assert phrase in doc, phrase


def test_word_positions():
    pe, tok = _pe(), ToyTokenizer()
    assert pe.word_positions(tok, "a cat riding a bicycle") == [[1], [2], [3, 4], [5], [6, 7]]
    assert pe.positions_of(tok, "a cat riding a bicycle", "a") == [1, 5]
    assert pe.positions_of(tok, "a cat riding a bicycle", ["bicycle", 1]) == [6, 7, 2]
    with pytest.raises(ValueError, match="not in the prompt"):
        pe.positions_of(tok, "a cat", "dog")


def test_replacement_mapper_equal_and_unequal_token_counts():
    pe, tok = _pe(), ToyTokenizer()
    assert np.array_equal(pe.replacement_mapper(tok, "a cat riding a bike", "a dog riding a bike"), np.eye(L))
    # 1 source token -> 2 target tokens: weight 1/2 each, later positions shifted by one, position 76 of the source unmapped
    M = pe.replacement_mapper(tok, "a cat rides", "a kitten rides")
    assert M[0, 0] == M[1, 1] == 1 and M[2, 2] == M[2, 3] == 0.5
    for k in range(3, 76):
        assert M[k, k + 1] == 1
    assert M.sum() == 2 + 1 + 73 and not M[76].any()
    # 2 source tokens -> 1: both map to it with weight 1, later positions shifted back, target position 76 maps to itself
    M = pe.replacement_mapper(tok, "a kitten rides", "a cat rides")
    assert M[2, 2] == M[3, 2] == 1
    for k in range(4, 77):
        assert M[k, k - 1] == 1
    assert M[76, 76] == 1 and M.sum() == 2 + 2 + 73 + 1
    # equal piece counts map one to one
    M = pe.replacement_mapper(tok, "a kitten", "a puppyy")
    assert M[2, 2] == M[3, 3] == 1 and M[2, 3] == 0
    with pytest.raises(ValueError, match="equal word counts"):
        pe.replacement_mapper(tok, "a cat", "a black cat")


def test_alignment_insertions_substitutions_ties():
    pe = _pe()
    assert pe.align([0, 1, 2, 3, 9], [0, 1, 7, 2, 3, 9]) == [0, 1, -1, 2, 3, 4]      # insertion
    assert pe.align([0, 1, 2, 3, 9], [0, 1, 8, 3, 9]) == [0, 1, 2, 3, 4]             # substitution (mismatch on the diagonal)
    assert pe.align([0, 5, 9], [0, 6, 7, 9]) == [0, -1, 1, 2]                        # tie: diagonal first, then the insertion
    tok = ToyTokenizer()
    mp, alpha = pe.refinement_map(tok, "a cat", "a red cat")
    assert list(alpha[:5]) == [1, 1, 0, 1, 1] and list(mp[:5]) == [0, 1, 2, 2, 3]
    assert np.array_equal(mp[5:], np.arange(5, L)) and (alpha[5:] == 1).all()


def test_equalizer_and_reweight():
    pe, tok = _pe(), ToyTokenizer()
    c = pe.equalizer(tok, "a fluffy cat", ["fluffy", "cat"], [2.0, 0.5])
    want = np.ones(L)
    want[[2, 3]] = 2.0
    want[4] = 0.5
    assert np.array_equal(c, want)
    ed = pe.reweight(tok, ["a fluffy cat", "a fluffy cat", "a fluffy cat"], "fluffy", 3.0)
    assert ed.n == 3 and not ed.has_beta and np.array_equal(ed.A[1], np.diag(np.where(np.arange(L) // 2 == 1, 3.0, 1.0)))
    with pytest.raises(ValueError, match="2 words and 1 values"):
        pe.equalizer(tok, "a fluffy cat", ["fluffy", "cat"], [2.0])


def test_builders_tables():
    pe, tok = _pe(), ToyTokenizer()
    ed = pe.replace(tok, ["a cat rides", "a dog rides", "a kitten rides"], cross_steps=0.8, self_steps=0.4,
                    blend_words=[["cat"], ["dog"], ["kitten"]], blend_start=0.5)
    assert ed.blend.shape == (3, L) and ed.blend[0, 2] == 1 and ed.blend[2, 2] == ed.blend[2, 3] == 1 and ed.blend.sum() == 4
    T = 10
    tab = ed.tables(T, cfg=True)
    assert tab['cross2'] is None and tab['cross'].shape == (T, 3, 6) and tab['cross'].dtype == np.int32
    ident = np.arange(6)
    for i in range(T):
        idx = T - 1 - i
        for name, window in (('cross', 8), ('self', 4)):
            t = tab[name][idx]
            for r in range(6):
                if r >= 4 and i < window:       # conditional rows of the targets: q, k of the source row 3
                    want = (3, 3, 6 + r - 4) if name == 'cross' else (3, 3, r)
                else:
                    want = (r, r, r)
                assert tuple(t[:, r]) == want, (name, i, r)
        assert tab['flags'][idx] == int(i >= 5)
    # without CFG the conditional rows start at 0
    t = ed.tables(4, cfg=False)['cross'][3]
    assert t[:, 0].tolist() == [0, 0, 0] and t[:, 1].tolist() == [0, 0, 3] and t[:, 2].tolist() == [0, 0, 4]
    assert np.array_equal(ed.tables(4, cfg=False)['cross'][0], np.broadcast_to(np.arange(3), (3, 3)))
    # refine: the second term of each target whose beta is not all zero reads its own q, k and ctx''
    rf = pe.refine(tok, ["a cat", "a red cat", "a cat"], cross_steps=0.5)
    assert rf.has_beta and rf.beta[0, 2] == 1 and not rf.beta[1].any()
    c2 = rf.tables(4, cfg=True)['cross2']
    assert tuple(c2[3][:, 4]) == (4, 4, 8) and (c2[3][2, [0, 1, 2, 3, 5]] == -1).all() and (c2[1] == -1).all()
    # no blend words: no flags
    assert not pe.replace(tok, ["a cat", "a dog"]).tables(5, True)['flags'].any()


def _softmax(s):
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


@pytest.mark.parametrize("kind", ["replace", "refine", "reweight"])
def test_factored_form_equals_p2p_on_probabilities(kind):
    """P_src V(A ctx) + P_tgt V(diag(beta) ctx) == P2P's edit of the probabilities times V(ctx), in fp64."""
    pe, tok = _pe(), ToyTokenizer()
    g = np.random.default_rng(5)
    prompts = {"replace": ["a cat riding a bicycle", "a kitten riding a bicycle"],
               "refine": ["a cat riding a bicycle", "a fluffy cat riding a red bicycle"],
               "reweight": ["a fluffy cat", "a fluffy cat"]}[kind]
    eq = (["riding"], [1.75]) if kind != "reweight" else None
    if kind == "replace":
        ed = pe.replace(tok, prompts, equalize=eq)
    elif kind == "refine":
        ed = pe.refine(tok, prompts, equalize=eq)
    else:
        ed = pe.reweight(tok, prompts, "fluffy", 2.5)
    h, N, C, d = 3, 11, 24, 8
    ctx = g.standard_normal((L, C))
    wv = g.standard_normal((C, h * d))
    V = lambda c: (c @ wv).reshape(L, h, d).transpose(1, 0, 2)          # [h, L, d]
    p_src, p_tgt = _softmax(g.standard_normal((h, N, L)) * 3), _softmax(g.standard_normal((h, N, L)) * 3)
    A, beta = ed.A[0].astype(np.float64), ed.beta[0].astype(np.float64)
    factored = p_src @ V(A @ ctx) + p_tgt @ V(beta[:, None] * ctx)
    c = pe.equalizer(tok, prompts[1], *(eq or ("fluffy", 2.5)))
    if kind == "replace":
        edited = np.einsum("hpw,wn->hpn", p_src, pe.replacement_mapper(tok, prompts[0], prompts[1])) * c
    elif kind == "refine":
        mp, alpha = pe.refinement_map(tok, prompts[0], prompts[1])
        assert (alpha == 0).any()
        edited = (alpha * p_src[:, :, mp] + (1 - alpha) * p_tgt) * c
    else:
        edited = p_src * c
    want = edited @ V(ctx)
    # A and beta are stored in fp32: the equalizer weights (1.75, 2.5) are exact there, the 1/t mapper weights too
    assert np.abs(factored - want).max() <= 1e-12 * np.abs(want).max(), np.abs(factored - want).max()


def test_prompt_edit_argument_checks():
    pe = _pe()
    A, beta = np.zeros((1, L, L)), np.zeros((1, L))
    with pytest.raises(ValueError, match="n >= 2"):
        pe.PromptEdit(np.zeros((0, L, L)), np.zeros((0, L)), 0.5, 0.5)
    with pytest.raises(ValueError, match="beta: expected"):
        pe.PromptEdit(A, np.zeros((2, L)), 0.5, 0.5)
    for k in ("cross_steps", "self_steps", "blend_start"):
        with pytest.raises(ValueError, match=k):
            pe.PromptEdit(A, beta, **{"cross_steps": 0.5, "self_steps": 0.5, k: 1.5})
    with pytest.raises(ValueError, match="blend: expected"):
        pe.PromptEdit(A, beta, blend=np.zeros((1, L)))
    with pytest.raises(ValueError, match="source and at least one target"):
        pe.replace(ToyTokenizer(), ["a cat"])
    assert [pe.quarter(s) for s in (64, 16, 62, 60, 1)] == [16, 4, 16, 15, 1]


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def _cinfo(n=3, typ="text", Lc=77, ed=None, scale=7.5):
    ci = {"type": typ, "conditioning": torch.zeros(n, Lc, 768), "unconditional_conditioning": torch.zeros(n, Lc, 768),
          "unconditional_guidance_scale": scale}
    if ed is not None:
        ci["prompt_edit"] = ed
    return ci


def test_refusals_before_any_device_work():
    """The fake model is on the CPU: a call that got past the checks would raise the sampler's 'no CPU path' RuntimeError."""
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    from lib.model_zoo.plms import PLMSSampler
    pe = _pe()
    ed = pe.replace(ToyTokenizer(), ["a cat", "a dog", "a fox"])
    shape = [3, 4, 8, 8]
    img = {"type": "image"}
    for S in (DDIMSampler(_fake_model()), DPMSolverSampler(_fake_model())):
        run = lambda x_info, cl, shp=shape: S.sample_multicontext(steps=5, shape=shp, x_info=x_info, c_info_list=cl, verbose=False) \
            if len(cl) > 1 else S.sample(steps=5, shape=shp, x_info=x_info, c_info=cl[0], verbose=False)
        for k, v in (("x0", torch.zeros(3, 4, 8, 8)), ("inpaint_mask", torch.ones(1, 1, 8, 8)), ("inversion", object())):
            with pytest.raises(ValueError, match=f"does not combine with '{k}'"):
                run(dict(img, **{k: v}), [_cinfo(ed=ed)])
        with pytest.raises(ValueError, match="text latent"):
            run({"type": "text"}, [_cinfo(ed=ed)], [3, 768])
        with pytest.raises(ValueError, match="must ride on a text context"):
            run(img, [_cinfo(), _cinfo(typ="image", Lc=257, ed=ed)])
        with pytest.raises(ValueError, match="conditioning batch of 3"):
            run(img, [_cinfo(n=2, ed=ed)])
        with pytest.raises(ValueError, match="conditioning batch of 3"):
            run(img, [_cinfo(ed=ed), _cinfo(n=2, typ="image", Lc=257)])
        with pytest.raises(ValueError, match="a batch of 3"):
            run(img, [_cinfo(ed=ed)], [2, 4, 8, 8])
        with pytest.raises(ValueError, match="'xt' must be"):
            run(dict(img, xt=torch.zeros(2, 4, 8, 8)), [_cinfo(ed=ed)])
        with pytest.raises(ValueError, match="one context may carry"):
            run(img, [_cinfo(ed=ed), _cinfo(ed=ed)])
        # accepted inputs reach the device stage
        for xt in (None, torch.zeros(1, 4, 8, 8), torch.zeros(3, 4, 8, 8)):
            with pytest.raises(RuntimeError, match="no CPU path"):
                run(img if xt is None else dict(img, xt=xt), [_cinfo(ed=ed), _cinfo(typ="image", Lc=257)])
    with pytest.raises(NotImplementedError, match="PLMSSampler has no prompt editing"):
        PLMSSampler(_fake_model()).sample(steps=5, shape=shape, x_info=img, c_info=_cinfo(ed=ed), verbose=False)
    S = DDIMSampler(_fake_model())
    S.make_schedule(5, verbose=False)
    x_info = {"type": "image", "x": torch.zeros(3, 4, 8, 8)}
    with pytest.raises(NotImplementedError, match="spans the walk"):
        S.p_sample_ddim(x_info, _cinfo(ed=ed), torch.zeros(3, dtype=torch.long), 4)
    with pytest.raises(NotImplementedError, match="spans the walk"):
        S.p_sample_ddim_multicontext(x_info, [_cinfo(ed=ed)], torch.zeros(3, dtype=torch.long), 4)


def test_items_attention_word_map_and_blend_reject_bad_arguments_without_gpu():
    """vdb_attention_bf16 with an item table, vdb_xattn_word_map_f32 and vdb_local_blend_f32 refuse bad arguments before any
    launch (the fake addresses are never dereferenced)."""
    from vdb200._lib import lib
    before = lib.vdb_launch_count()
    at = dict(q=0x100000, k=0x200000, vt=0x300000, out=0x400000, items=0x500000, idx=0x600000, Bq=4, Bkv=6, acc=1, d=40)

    def attn(**kw):
        a = dict(at, **kw)
        return lib.vdb_attention_bf16(a["q"], 1280, 0, a["k"], 1280, 0, a["vt"], 512, a["out"], 1280, 4, 8, 64, 77, 0, 80,
                                      a["d"], 0.125, 0, None, a["Bq"], a["Bkv"], a["items"], a["idx"], a["acc"], None)

    for k in ("items", "idx"):
        assert attn(**{k: None}) == 1 and b"attention: items and step_idx" in lib.vdb_last_error(), k
        assert attn(**{k: at[k] + 2}) == 1 and b"4-byte aligned" in lib.vdb_last_error(), k
    for k in ("Bq", "Bkv"):
        assert attn(**{k: 0}) == 1 and b"Bq and Bkv" in lib.vdb_last_error(), k
    # Bq, Bkv, step_idx and accumulate belong to the table: each one alone, without items, is refused
    none = dict(items=None, idx=None, Bq=0, Bkv=0, acc=0)
    for k in ("Bq", "Bkv", "idx", "acc"):
        assert attn(**dict(none, **{k: at[k]})) == 1 and b"items and step_idx" in lib.vdb_last_error(), k
    for k in ("q", "k", "vt", "out"):
        assert attn(**{k: None}) == 1 and b"attention: null" in lib.vdb_last_error(), k
    assert attn(d=44) == 1 and b"multiples of 8" in lib.vdb_last_error()

    wm = dict(q=0x100000, k=0x200000, w=0x300000, map=0x400000, n=3, row0=3, H=8, N=256, L=77, kv=80, d=160)

    def wmap(**kw):
        a = dict(wm, **kw)
        return lib.vdb_xattn_word_map_f32(a["q"], 1536, a["k"], 1536, a["w"], a["map"], a["n"], a["row0"], a["H"], a["N"], a["L"],
                                          a["kv"], a["d"], 0.08, None)

    for k in ("q", "k", "w", "map"):
        assert wmap(**{k: None}) == 1 and b"xattn_word_map: null" in lib.vdb_last_error(), k
        assert wmap(**{k: wm[k] + 2}) == 1 and b"4-byte aligned" in lib.vdb_last_error(), k
    for k in ("n", "H", "N", "L"):
        assert wmap(**{k: 0}) == 1 and b"empty" in lib.vdb_last_error(), k
    assert wmap(row0=-1) == 1
    assert wmap(kv=72) == 1 and b"kv_bstride >= L" in lib.vdb_last_error()
    assert wmap(L=81, kv=88) == 3 and b"at most 80 keys" in lib.vdb_last_error()
    assert wmap(d=168) == 3
    assert wmap(map=wm["w"] + 4 * 8) == 1 and b"overlaps" in lib.vdb_last_error()

    bl = dict(x=0x100000, dup=0x200000, map=0x300000, flags=0x400000, idx=0x500000, n=3, H=64, W=64, C=4, h=16, w=16, thr=0.3)

    def blend(**kw):
        a = dict(bl, **kw)
        return lib.vdb_local_blend_f32(a["x"], a["dup"], a["map"], a["flags"], a["idx"], a["n"], a["H"], a["W"], a["C"], a["h"],
                                       a["w"], a["thr"], None)

    for k in ("x", "map", "flags", "idx"):
        assert blend(**{k: None}) == 1 and b"local_blend: null" in lib.vdb_last_error(), k
    for k in ("x", "dup", "map", "flags", "idx"):
        assert blend(**{k: bl[k] + 2}) == 1 and b"4-byte aligned" in lib.vdb_last_error(), k
    for k in ("n", "H", "W", "C", "h", "w"):
        assert blend(**{k: 1 if k == "n" else 0}) == 1 and b"empty" in lib.vdb_last_error(), k
    assert blend(h=65, w=64) == 1 and b"at most 4096" in lib.vdb_last_error()
    for v in (float("nan"), float("inf")):
        assert blend(thr=v) == 1 and b"finite" in lib.vdb_last_error()
    for k, addr in (("map", bl["x"] + 4 * 100), ("dup", bl["x"] + 4 * 4), ("map", bl["dup"] - 4)):
        assert blend(**{k: addr}) == 1 and b"overlap" in lib.vdb_last_error(), (k, addr)
    assert lib.vdb_launch_count() == before
