"""Prompt-to-Prompt on the GPU (lib/model_zoo/prompt_edit.py): vdb_attention_bf16 with an item table per element against fp64
at every instantiation (with random tables, skips and accumulation) and bitwise against the plain form under the identity table,
vdb_xattn_word_map_f32 against fp64, vdb_local_blend_f32 bitwise against its fp32 restatement; on the mini UNet the edited DDIM
and DPM-Solver++ walks against oracle/prompt_edit_oracle.py; and the invariants: the source row and a zero-window edit equal
the unedited batch bit for bit, the graph equals eager, a second call replays the cached graph, and the launches per step."""
import numpy as np
import pytest
import torch

from oracle import prompt_edit_oracle as P
from test_parity_gpu import build_net
from test_prompt_edit import ToyTokenizer

pytestmark = pytest.mark.gpu
DEV = "cuda"
L = 77
SCALE = 3.0


def _bf(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV).to(torch.bfloat16)


def _operands(g, Bq, Bkv, H, d, Nq, kvb):
    """Q [Bq*Nq, H*DK], K [Bkv*kvb, H*DK], V^T [H*DVP, Bkv*kvb] bf16 with zero head pads, and their fp64 values."""
    from vdb200 import ops
    DK, DVP = ops.attention_pads(d)
    q = np.zeros((Bq * Nq, H, DK)); q[:, :, :d] = g.standard_normal((Bq * Nq, H, d))
    k = np.zeros((Bkv * kvb, H, DK)); k[:, :, :d] = g.standard_normal((Bkv * kvb, H, d))
    v = np.zeros((H, DVP, Bkv * kvb)); v[:, :d] = g.standard_normal((H, d, Bkv * kvb))
    tq, tk, tv = _bf(q.reshape(Bq * Nq, -1)), _bf(k.reshape(Bkv * kvb, -1)), _bf(v.reshape(H * DVP, -1))
    f = lambda t, s: t.float().cpu().double().numpy().reshape(s)
    return tq, tk, tv, f(tq, q.shape)[:, :, :d], f(tk, k.shape)[:, :, :d], f(tv, v.shape)[:, :d]


def _ref(q, k, v, bq, bk, bv, Nq, Nk, kvb, scale):
    """fp64 attention of one output item -> [Nq, H, d]."""
    qb = q[bq * Nq:(bq + 1) * Nq]                       # [Nq, H, d]
    kb = k[bk * kvb:bk * kvb + Nk]                      # [Nk, H, d]
    vb = v[:, :, bv * kvb:bv * kvb + Nk]                # [H, d, Nk]
    s = np.einsum("phc,jhc->hpj", qb, kb) * scale
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    return np.einsum("hpj,hcj->phc", p, vb)


@pytest.mark.parametrize("d", [8, 16, 32, 40, 64, 80, 160])
def test_attention_with_items_per_element(d):
    from vdb200 import ops
    g = np.random.default_rng(d)
    B, Bq, Bkv, H, Nq, Nk, kvb = 4, 5, 7, 2, 200, 77, 80
    tq, tk, tv, q, k, v = _operands(g, Bq, Bkv, H, d, Nq, kvb)
    scale = d ** -0.5
    items = np.stack([np.stack([g.integers(0, Bq, B), g.integers(0, Bkv, B), g.integers(0, Bkv, B)]) for _ in range(3)]).astype(np.int32)
    items[1, 2, 2] = -1                                                     # row 1 skips item 2
    ti = torch.from_numpy(items).to(DEV)
    for acc in (False, True):
        prev = g.standard_normal((B * Nq, H * d)).astype(np.float32)
        out = _bf(prev)
        prev64 = out.float().cpu().double().numpy()
        ops.attention(tq, tk, tv, out, B, H, Nq, Nk, d, kv_bstride=kvb, items=ti,
                      step_idx=torch.tensor([1], dtype=torch.int32, device=DEV), Bq=Bq, Bkv=Bkv, accumulate=acc)
        got = out.float().cpu().double().numpy()
        for b in range(B):
            rows = slice(b * Nq, (b + 1) * Nq)
            bq, bk, bv = items[1, :, b]
            if bv < 0:
                assert np.array_equal(got[rows], prev64[rows]), "a skipped item is not written"
                continue
            want = _ref(q, k, v, bq, bk, bv, Nq, Nk, kvb, scale).reshape(Nq, H * d) + (prev64[rows] if acc else 0)
            err = np.abs(got[rows] - want).max()
            assert err <= 2e-2 * np.abs(want).max() + 1e-3, (d, acc, b, err)


@pytest.mark.parametrize("d", [8, 40, 64, 80, 160])
def test_identity_items_table_equals_plain_attention(d):
    from vdb200 import ops
    g = np.random.default_rng(100 + d)
    B, H, Nq, Nk, kvb = 3, 2, 256, 77, 80
    tq, tk, tv, *_ = _operands(g, B, B, H, d, Nq, kvb)
    plain = torch.empty(B * Nq, H * d, dtype=torch.bfloat16, device=DEV)
    ops.attention(tq, tk, tv, plain, B, H, Nq, Nk, d, kv_bstride=kvb)
    ident = torch.arange(B, dtype=torch.int32, device=DEV).view(1, 1, B).repeat(2, 3, 1).contiguous()
    out = torch.empty_like(plain)
    ops.attention(tq, tk, tv, out, B, H, Nq, Nk, d, kv_bstride=kvb, items=ident,
                  step_idx=torch.tensor([1], dtype=torch.int32, device=DEV))
    assert torch.equal(out, plain)


@pytest.mark.parametrize("d,H,N", [(8, 8, 16), (40, 8, 256), (160, 8, 256), (80, 2, 37)])
def test_word_map_against_fp64(d, H, N):
    from vdb200 import ops
    g = np.random.default_rng(d + N)
    n, B, Bkv, kvb, row0 = 3, 6, 8, 80, 3
    tq, tk, _, q, k, _ = _operands(g, B, Bkv, H, d, N, kvb)
    w = (g.random((n, L)) < 0.1).astype(np.float32)
    m0 = g.random((n, N)).astype(np.float32)
    out = torch.from_numpy(m0).to(DEV)
    ops.xattn_word_map(tq, tk, torch.from_numpy(w).to(DEV), out, row0, H, N, L, d, kv_bstride=kvb)
    got = out.cpu().numpy()
    want = m0.astype(np.float64).copy()
    for r in range(n):
        qb, kb = q[(row0 + r) * N:(row0 + r + 1) * N], k[(row0 + r) * kvb:(row0 + r) * kvb + L]
        s = np.einsum("phc,jhc->hpj", qb, kb) * d ** -0.5
        p = np.exp(s - s.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        want[r] += (p * w[r]).sum(axis=(0, 2))
    assert np.abs(got - want).max() <= 1e-5 * H, np.abs(got - want).max()
    again = torch.from_numpy(m0).to(DEV)
    ops.xattn_word_map(tq, tk, torch.from_numpy(w).to(DEV), again, row0, H, N, L, d, kv_bstride=kvb)
    assert np.array_equal(again.cpu().numpy(), got), "bit-reproducible"


def _blend_f32(x, wmap, h, w, thr):
    """vdb_local_blend_f32 restated in fp32 numpy."""
    n, H, W, C = x.shape
    m = wmap.reshape(n, h, w)
    pad = np.pad(m, ((0, 0), (1, 1), (1, 1)), constant_values=-np.inf)
    pooled = np.max([pad[:, dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)], axis=0)
    mx = pooled.reshape(n, -1).max(1)
    ys, xs = (np.arange(H) * h) // H, (np.arange(W) * w) // W
    up = pooled[:, ys][:, :, xs]
    with np.errstate(invalid="ignore", divide="ignore"):
        mask = (mx[:, None, None] > 0) & ((up / mx[:, None, None]).astype(np.float32) > np.float32(thr))
    out = x.copy()
    for b in range(1, n):
        out[b] = np.where((mask[b] | mask[0])[:, :, None], x[b], x[0])
    return out


@pytest.mark.parametrize("n,H,W,h,w", [(3, 16, 16, 4, 4), (4, 64, 64, 16, 16), (2, 30, 22, 8, 6)])
def test_local_blend_bitwise(n, H, W, h, w):
    from vdb200 import ops
    g = np.random.default_rng(n * H + w)
    C, thr = 4, 0.3
    x = g.standard_normal((n, H, W, C)).astype(np.float32)
    wmap = g.random((n, h * w)).astype(np.float32) ** 3
    wmap[n - 1] = 0.0                                       # an all-zero map: that mask is false everywhere
    flags = torch.tensor([0, 1], dtype=torch.int32, device=DEV)
    for idx in (0, 1):
        tx = torch.from_numpy(x).to(DEV)
        dup = torch.full_like(tx, float("nan"))
        ops.local_blend(tx, torch.from_numpy(wmap).to(DEV), flags, torch.tensor([idx], dtype=torch.int32, device=DEV), h, w, thr,
                        x_dup=dup)
        if idx == 0:
            assert torch.equal(tx.cpu(), torch.from_numpy(x)) and torch.isnan(dup).all(), "flag 0 leaves x alone"
            continue
        want = _blend_f32(x, wmap, h, w, thr)
        assert np.array_equal(tx.cpu().numpy(), want)
        assert np.array_equal(dup.cpu().numpy()[1:], want[1:]) and torch.isnan(dup[0]).all()


# ---- the walks on the mini UNet -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd


PROMPTS = {"replace": ["a cat riding a bike", "a kitten riding a bike", "a dog riding a bike"],
           "refine": ["a cat riding a bike", "a fluffy cat riding a bike", "a cat riding a red bike"],
           "reweight": ["a fluffy cat", "a fluffy cat", "a fluffy cat"]}
BLEND = {"replace": [["cat"], ["kitten"], ["dog"]], "refine": [["cat"], ["cat"], ["bike"]],
         "reweight": [["cat"], ["cat"], ["cat"]]}


def _edit(kind, blend, cross=0.6, self_=0.4, blend_start=0.0, threshold=0.8):
    from lib.model_zoo import prompt_edit as pe
    tok, pr = ToyTokenizer(), PROMPTS[kind]
    bw = BLEND[kind] if blend else None
    if kind == "replace":
        ed = pe.replace(tok, pr, cross, self_, blend_words=bw, equalize=(["riding"], [1.5]), blend_start=blend_start,
                        threshold=threshold)
        comp = dict(M=np.stack([pe.replacement_mapper(tok, pr[0], p) for p in pr[1:]]))
        c = np.stack([pe.equalizer(tok, p, ["riding"], [1.5]) for p in pr[1:]])
    elif kind == "refine":
        ed = pe.refine(tok, pr, cross, self_, blend_words=bw, blend_start=blend_start, threshold=threshold)
        maps = [pe.refinement_map(tok, pr[0], p) for p in pr[1:]]
        comp = dict(mp=np.stack([m for m, _ in maps]), alpha=np.stack([a for _, a in maps]))
        c = np.ones((2, L))
    else:
        ed = pe.reweight(tok, pr, "fluffy", [2.0], cross, self_, blend_words=bw, blend_start=blend_start)
        comp, c = {}, np.stack([pe.equalizer(tok, p, "fluffy", 2.0) for p in pr[1:]])
        c[1] = 1.0
        ed = pe.PromptEdit(np.stack([ed.A[0], np.eye(L)]), ed.beta, cross, self_, ed.blend, threshold, blend_start)
    return ed, comp, c


def _contexts(n, multi, g):
    """The golden mini prompt pair, the conditional rows perturbed per prompt (a well-conditioned walk at CFG 3)."""
    from oracle.make_golden import golden_inputs
    gi = golden_inputs("mini")
    ct, ut = gi["c"] + 0.2 * torch.randn(n, L, 768, generator=g), gi["u"].repeat(n, 1, 1)
    ci = lambda c, u, typ, r, ed: dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                                        "unconditional_guidance_scale": SCALE, "ratio": r}, **({"prompt_edit": ed} if ed else {}))
    if multi:
        cim, uim = torch.randn(n, 257, 768, generator=g) * 0.5, torch.zeros(n, 257, 768)
        return [ct, cim], [ut, uim], dict(c_types=("text", "image"), ratios=[0.7, 0.3]), \
            lambda ed: [ci(ct, ut, "text", 0.7, ed), ci(cim, uim, "image", 0.3, None)]
    return [ct], [ut], dict(c_types=("text",), ratios=None), lambda ed: [ci(ct, ut, "text", 1.0, ed)]


def _sample(S, steps, shape, x_info, cl):
    kw = dict(steps=steps, shape=shape, x_info=dict(x_info), verbose=False, eta=0.)
    with torch.no_grad():
        return (S.sample_multicontext(c_info_list=cl, **kw) if len(cl) > 1 else S.sample(c_info=cl[0], **kw))[0]


def _sampler(net, kind, **kw):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return DDIMSampler(net, **kw) if kind == "ddim" else DPMSolverSampler(net, order=2, **kw)


def _fidelity(x, ref):
    x, ref = x.cpu().double().flatten(), ref.double().flatten()
    return torch.nn.functional.cosine_similarity(x, ref, dim=0).item(), (x - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("edit,blend,multi,sampler", [("replace", True, False, "ddim"), ("refine", False, True, "ddim"),
                                                      ("reweight", True, True, "dpmpp"), ("replace", False, True, "dpmpp"),
                                                      ("refine", True, False, "dpmpp"), ("reweight", False, False, "ddim")])
def test_edited_walk_vs_oracle(mini, edit, blend, multi, sampler):
    """A walk from pure noise on the random-weight mini UNet amplifies bf16 rounding (x reaches ~20 in six steps), so the edited
    walk is held to the fidelity the unedited walk of the same inputs reaches against the same oracle, and the edit's effect on
    the device (edited minus unedited) must point where the oracle's does: cosine 0.79 - 0.87 on an H100 for these cases, where
    an unrelated perturbation gives about 0.  The kernels themselves are checked per element above."""
    net, sd = mini
    g = torch.Generator().manual_seed(53)
    n, C, H, W, steps = 3, 4, 16, 16, 6
    ed, comp, c = _edit(edit, blend)
    conds, unconds, okw, cl = _contexts(n, multi, g)
    xt = torch.randn(1, C, H, W, generator=g)
    x_info = {"type": "image", "xt": xt.expand(n, C, H, W).contiguous().to(DEV)}
    x = _sample(_sampler(net, sampler), steps, [n, C, H, W], x_info, cl(ed))
    plain = _sample(_sampler(net, sampler), steps, [n, C, H, W], x_info, cl(None))
    ctl = P.P2P(n, edit, steps, ed.cross_steps, ed.self_steps, c, H, W, w=ed.blend, threshold=ed.threshold, **comp)
    ref = P.sample(sd, ctl, xt.expand(n, C, H, W), conds, unconds, steps, sampler=sampler, scale=SCALE, model_channels=64, **okw)
    off = P.P2P(n, edit, steps, 0.0, 0.0, c, H, W, **comp)
    ref0 = P.sample(sd, off, xt.expand(n, C, H, W), conds, unconds, steps, sampler=sampler, scale=SCALE, model_channels=64, **okw)
    what = f"{edit} {'blend' if blend else 'no blend'} {'dual' if multi else 'single'} {sampler}"
    cos, rel = _fidelity(x, ref)
    cos0, rel0 = _fidelity(plain, ref0)
    d_dev, d_ref = (x - plain).cpu().double()[1:].flatten(), (ref - ref0).double()[1:].flatten()
    agree = torch.nn.functional.cosine_similarity(d_dev, d_ref, dim=0).item()
    print(f"[p2p] {what}: edited cos {cos:.6f} max rel err {rel:.4f}; unedited cos {cos0:.6f} max rel err {rel0:.4f}; "
          f"edit effect |d| {d_ref.norm().item():.3g}, device vs oracle cos {agree:.4f}")
    assert cos >= min(0.995, cos0 - 0.002) and rel <= 1.5 * rel0 + 0.02, what
    assert agree >= 0.7, what
    assert torch.equal(x[0], plain[0]), "the source row is never edited"


@pytest.mark.parametrize("sampler", ["ddim", "dpmpp"])
def test_invariants(mini, sampler):
    net, _ = mini
    g = torch.Generator().manual_seed(59)
    n, C, H, W, steps = 3, 4, 16, 16, 6
    shape = [n, C, H, W]
    _, _, _, cl = _contexts(n, False, g)
    xt = {"type": "image", "xt": torch.randn(1, C, H, W, generator=g).expand(n, C, H, W).contiguous().to(DEV)}
    S0 = _sampler(net, sampler)
    plain = _sample(S0, steps, shape, xt, cl(None))
    ed, _, _ = _edit("replace", True)
    Se = _sampler(net, sampler)
    edited = _sample(Se, steps, shape, xt, cl(ed))
    assert torch.equal(edited[0], plain[0]), "the source row is never edited"
    assert not torch.equal(edited[1], plain[1])
    zero, _, _ = _edit("replace", False, cross=0.0, self_=0.0)
    Sz = _sampler(net, sampler)
    assert torch.equal(_sample(Sz, steps, shape, xt, cl(zero)), plain), "empty windows, no blend: the unedited batch"
    # launches per step: the word maps of the five 1/4-side cross layers and the blend; refinement adds one per cross layer
    print(f"[p2p] {sampler} launches per step: plain {S0.last_step_launches}, zero windows {Sz.last_step_launches}, "
          f"replace + blend {Se.last_step_launches}")
    assert Sz.last_step_launches == S0.last_step_launches
    assert Se.last_step_launches == S0.last_step_launches + 5 + 1
    rf, _, _ = _edit("refine", False)
    Sr = _sampler(net, sampler)
    _sample(Sr, steps, shape, xt, cl(rf))
    assert Sr.last_step_launches == S0.last_step_launches + 16, Sr.last_step_launches
    # graph against eager
    eager = _sample(_sampler(net, sampler, use_cuda_graph=False), steps, shape, xt, cl(ed))
    assert torch.equal(eager, edited), "graph path must be bit-identical to the eager path"
    # a second call on new prompts, tables and noise replays the cached graph and equals a fresh sampler
    graph = next(iter(Se._graphs.values()))[0]
    _, _, _, cl2 = _contexts(n, False, g)
    ed2, _, _ = _edit("replace", True, cross=0.4, self_=0.2, blend_start=0.3)
    Se.last_step_launches = None
    torch.manual_seed(3)
    again = _sample(Se, steps, shape, {"type": "image"}, cl2(ed2))
    assert next(iter(Se._graphs.values()))[0] is graph and Se.last_step_launches is None, "no eager step, no capture"
    torch.manual_seed(3)
    fresh = _sample(_sampler(net, sampler), steps, shape, {"type": "image"}, cl2(ed2))
    assert torch.equal(again, fresh)
    assert not torch.equal(again, edited)
    # without 'xt' every row starts from one draw: the unedited walk of equal prompts gives equal rows
    _, _, _, cl3 = _contexts(1, False, g)
    same = [dict(ci, conditioning=ci["conditioning"].expand(n, L, 768), unconditional_conditioning=ci["unconditional_conditioning"]
                 .expand(n, L, 768)) for ci in cl3(None)]
    zero3, _, _ = _edit("reweight", False, cross=0.0, self_=0.0)
    same[0]["prompt_edit"] = zero3
    out = _sample(_sampler(net, sampler), steps, shape, {"type": "image"}, same)
    assert torch.equal(out[1], out[0]) and torch.equal(out[2], out[0])
