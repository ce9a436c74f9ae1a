"""Repetition penalty and no-repeat n-gram bans of the text decoder on the GPU: vdb_textdec_repetition per element against the
numpy oracle (oracle/text_repetition_oracle.py) bitwise; both knobs off leave the decoder exactly as it is; a full-size decode
whose every step's recorded logits are the oracle's edit of the teacher-forced raw logits and whose every draw is the oracle's
pick; beam search against text_beam_oracle over processed logits; graph replay against eager; and net.vae_decode(x, 'text',
repetition_penalty=..., no_repeat_ngram_size=...) through the public surface.

Exemptions, as in test_text_filter_gpu / test_text_beam_gpu: a draw may differ from the oracle's when its uniform lies within 1e-6
of a step of the oracle's CDF (fp32 exp against fp64) or, with a nucleus cut, when it is the oracle's pick with top_p moved by 1e-5;
a beam selection whose fp64 margin is below 1e-12 may go either way, and such a latent is not compared afterwards."""
import json

import numpy as np
import pytest
import torch

from lib.model_zoo.optimus import decode_plan
from oracle.text_beam_oracle import BeamState, log_softmax64
from oracle.text_repetition_oracle import has_repeated_ngram, process, processed_beam_search, processed_pick

pytestmark = pytest.mark.gpu

DEV = "cuda"
EOS, BOS = 50259, 50258
MAX_LEN = 30
VFULL = 50260
NEAR_P = 1e-5
NEAR_BEAM = 1e-12


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def run_kernel(logits, tokens, done, s, penalty, n, pad=5):
    """ops.textdec_repetition on a device copy whose rows are views of rows pad floats wider -> (edited logits, launches)"""
    from vdb200 import ops
    R, V = logits.shape
    buf = torch.full((R, V + pad), 7.5)
    buf[:, :V] = torch.from_numpy(logits)
    buf = buf.to(DEV)
    tok = torch.from_numpy(np.ascontiguousarray(tokens)).to(torch.int32).to(DEV)
    dn = torch.from_numpy(np.ascontiguousarray(done)).to(torch.int32).to(DEV)
    n0 = ops.launch_count()
    ops.textdec_repetition(buf[:, :V], tok, dn, torch.tensor([s], dtype=torch.int32, device=DEV), penalty, n)
    launches = ops.launch_count() - n0
    out = buf.cpu().numpy()
    assert (out[:, V:] == 7.5).all(), "the padding between rows must stay untouched"
    return out[:, :V], launches


@pytest.mark.parametrize("V", [37, VFULL])
@pytest.mark.parametrize("R", [1, 5, 16])
def test_kernel_matches_the_oracle_bitwise(R, V):
    rng = np.random.default_rng(1000 * R + V)
    logits = (rng.standard_normal((R, V)) * 3).astype(np.float32)
    logits[:, :8] = np.array([0.0, -0.0, 3e38, -3e38, 1e-40, -1e-40, 1.0, -1.0], np.float32)
    tokens = np.empty((R, 33), np.int64)
    for r in range(R):
        kind = r % 4
        tokens[r] = (rng.integers(0, 6, 33) if kind == 0 else np.resize([3, 1, 4], 33) if kind == 1 else
                     rng.integers(-3, V + 3, 33) if kind == 2 else rng.integers(0, 9, 33))
    tokens[:, 0] = BOS                                          # outside [0, V) at V = 37
    tokens[:, 7] = -1
    tokens[:, 11] = V
    done = (rng.random(R) < 0.25).astype(np.int32)
    if R > 1:
        done[1] = 1
    cases = 0
    for s in (0, 1, 2, 3, 5, 17, 29, 31, 32):
        for n in (0, 1, 2, 3, 4, 30, 33):
            for p in (1.0, 0.5, 1.2, 3.0):
                got, launches = run_kernel(logits, tokens, done, s, p, n)
                want = logits if s + 1 >= 33 else process(logits, tokens, s, done, p, n)   # s + 1 >= ldt: nothing
                assert np.array_equal(_bits(got), _bits(want)), (R, V, s, n, p)
                assert launches == (0 if (p == 1.0 and n == 0) else 1)
                cases += 1
    print(f"[repetition] R{R} V{V}: {cases} cases bitwise equal to the oracle")


@pytest.fixture(scope="module")
def full():
    from test_text_decode_gpu import build_decoder
    return build_decoder(12, seed=11)


def latents(n, seed):
    return torch.randn(n, 768, generator=torch.Generator().manual_seed(seed)) * 3.0


def _same_beams(a, b):
    return len(a) == len(b) and all(len(x) == len(y) and all(torch.equal(p[0], q[0]) and p[1] == q[1] and p[2] == q[2]
                                                             for p, q in zip(x, y)) for x, y in zip(a, b))


def test_processors_off_are_the_existing_path(full):
    from vdb200 import ops
    m, _ = full
    z = latents(4, 31).to(DEV)
    u = torch.rand(4, 28, generator=torch.Generator().manual_seed(32), dtype=torch.float64).to(DEV)
    base_rows, base_rec = m.decode_ids(z, uniforms=u, return_logits=True)
    for kw in (dict(repetition_penalty=1.0, no_repeat_ngram_size=0), dict(repetition_penalty=1, no_repeat_ngram_size=0)):
        rows, rec = m.decode_ids(z, uniforms=u, return_logits=True, **kw)
        assert all(torch.equal(a, b) for a, b in zip(base_rows, rows)) and torch.equal(base_rec, rec), kw
        torch.manual_seed(3)
        a = m.decode_ids(z)
        torch.manual_seed(3)
        assert all(torch.equal(x, y) for x, y in zip(a, m.decode_ids(z, **kw))), kw
        assert _same_beams(m.decode_beams(z, 4), m.decode_beams(z, 4, **kw)), kw
    # launches: per step 64 (sampling) / 65 (beams) with both off, one more with either on; a whole eager decode likewise
    p = m.packed()
    for draw, K, R, off in (("seed", 0, 4, 64), ("beam", 4, 16, 65)):
        st = m._state(R, z.device)
        for (rp, nr), want in (((1.0, 0), off), ((1.3, 0), off + 1), ((1.0, 2), off + 1), ((1.3, 2), off + 1)):
            st.step.zero_()
            n0 = ops.launch_count()
            m._step(st, p, decode_plan(draw, 1.0, EOS, MAX_LEN, num_beams=K, repetition_penalty=rp, no_repeat_ngram_size=nr))
            assert ops.launch_count() - n0 == want, (draw, rp, nr)
    counts = []
    for kw in ({}, dict(repetition_penalty=1.0, no_repeat_ngram_size=0), dict(repetition_penalty=1.3, no_repeat_ngram_size=2)):
        n0 = ops.launch_count()
        m.decode_ids(z, eos_token=-1, graph=False, **kw)                   # <EOS> never drawn: all 28 steps run
        counts.append(ops.launch_count() - n0)
    assert counts[0] == counts[1] and counts[2] == counts[0] + 28, counts


def _pick_ok(tok, raw, h, s, rp, nr, temperature, top_k, top_p, u):
    """-> 0 if tok is the oracle's pick, 1 if it differs within an exemption; asserts otherwise"""
    pick, near, _ = processed_pick(raw, h, s, rp, nr, temperature, top_k, top_p, torch.tensor([u], dtype=torch.float64))
    if tok == int(pick[0]):
        return 0
    ok = float(near[0]) < 1e-6
    if 0.0 < top_p < 1.0:
        for q in (top_p - NEAR_P, min(top_p + NEAR_P, 1.0 - 1e-9)):
            ok |= tok == int(processed_pick(raw, h, s, rp, nr, temperature, top_k, q, torch.tensor([u], dtype=torch.float64))[0][0])
    assert ok, (s, tok, int(pick[0]), float(near[0]))
    return 1


@pytest.mark.parametrize("top_k,top_p,temperature", [(0, 0.0, 1.0), (40, 0.9, 0.7)])
def test_full_size_decode_follows_the_oracle(full, top_k, top_p, temperature):
    """penalty 1.3 and n = 2 with given uniforms: every recorded step is oracle.process of the teacher-forced raw logits of the
    produced prefix, bitwise; every draw is the oracle's pick with the same uniform; no row repeats a 2-gram."""
    m, _ = full
    rp, nr = 1.3, 2
    z = latents(4, 17)
    u = torch.rand(4, 28, generator=torch.Generator().manual_seed(18), dtype=torch.float64)
    rows, rec = m.decode_ids(z.to(DEV), temperature=temperature, uniforms=u.to(DEV), return_logits=True, top_k=top_k, top_p=top_p,
                             repetition_penalty=rp, no_repeat_ngram_size=nr)
    rec = rec.cpu().numpy()
    ids = torch.full((4, max(len(r) for r in rows)), EOS, dtype=torch.long)
    for r, row in enumerate(rows):
        ids[r, :len(row)] = row
    tf = m.teacher_forced_logits(z.to(DEV), ids).cpu().numpy()            # raw logits: teacher forcing takes no processors
    draws = exempt = edited = 0
    for r, row in enumerate(rows):
        h = row.numpy()
        assert h[0] == BOS and h[-1] == EOS and len(h) <= MAX_LEN, h
        assert not has_repeated_ngram(h, nr), h
        for s in range(min(len(h) - 1, rec.shape[0])):
            want = process(tf[r, s][None], h[None], s, None, rp, nr)[0]
            assert np.array_equal(_bits(rec[s, r]), _bits(want)), (r, s)
            edited += int((_bits(want) != _bits(tf[r, s])).sum())
            exempt += _pick_ok(int(h[s + 1]), tf[r, s], h, s, rp, nr, temperature, top_k, top_p, float(u[r, s]))
            draws += 1
    print(f"[repetition] full decode top_k {top_k} top_p {top_p}: {draws} steps, {edited} logits edited, {exempt} exempt draws, "
          f"lengths {[len(r) for r in rows]}")
    assert edited > draws and exempt <= draws // 50


@pytest.mark.parametrize("rp,nr", [(1.0, 2), (1.2, 3)])
def test_beam_plan_search_follows_the_oracle(full, rp, nr):
    m, _ = full
    n, K, temperature = 4, 4, 1.0
    z = latents(n, 25)
    plan = decode_plan("beam", temperature, EOS, record=True, num_beams=K, repetition_penalty=rp, no_repeat_ngram_size=nr)
    out, st, ran = m._beam_group(z.to(DEV), plan, 1.0, 1.0)
    rec, trace = st.record[:ran].cpu().numpy(), st.trace[:ran].cpu().numpy()
    zr = z.repeat_interleave(K, 0).to(DEV)
    raw = {}

    def raw_fn(s, hist):
        raw[s] = m.teacher_forced_logits(zr, torch.from_numpy(hist).long())[:, s].cpu().numpy()
        return raw[s]
    seen = dict(done=np.zeros(n * K, bool), diverged=set(), steps=0)

    def on_step(s, logits, new, wtrace, margins):
        for i in range(n):
            if margins[i] < NEAR_BEAM:
                print(f"[repetition] beam n{nr} step {s} latent {i}: oracle margin {margins[i]:.3g}, not compared from here on")
                seen["diverged"].add(i)
            if i in seen["diverged"]:
                continue
            for r in range(i * K, (i + 1) * K):               # recorded: the edited logits of live rows, raw ones of finished
                want = raw[s][r] if seen["done"][r] else logits[r]
                assert np.array_equal(_bits(rec[s, r]), _bits(want)), (s, r)
            rows = slice(i * K, (i + 1) * K)
            assert np.array_equal(trace[s, rows, :2], wtrace[rows, :2]), (s, i, trace[s, rows], wtrace[rows])
            a, b = trace[s, rows, 2], wtrace[rows, 2]
            assert ((a == b) | (np.abs(a - b) <= NEAR_BEAM * np.abs(b))).all(), (s, i, a, b)
        seen["done"] = new.done.copy()
        seen["steps"] += 1

    want, _ = processed_beam_search(raw_fn, n, K, BOS, EOS, MAX_LEN, temperature, rp, nr, on_step=on_step)
    assert seen["steps"] <= ran
    hyps = []
    for i in range(n):
        for j, (ids, sc, nm) in enumerate(out[i]):
            assert not has_repeated_ngram(ids.tolist(), nr), (i, ids)
            hyps.append((i, ids, sc))
            if i not in seen["diverged"]:
                wids, wsc, _ = want[i][j]
                assert ids.tolist() == wids.tolist() and abs(sc - wsc) <= NEAR_BEAM * abs(wsc), (i, j)
    # the returned scores re-score from the processed teacher-forced logits of each hypothesis
    ids = torch.full((len(hyps), max(len(h) for _, h, _ in hyps)), EOS, dtype=torch.long)
    for r, (_, h, _) in enumerate(hyps):
        ids[r, :len(h)] = h
    tf = m.teacher_forced_logits(z[[i for i, _, _ in hyps]].to(DEV), ids).cpu().numpy()
    for r, (_, h, sc) in enumerate(hyps):
        nsc = min(len(h) - 1, MAX_LEN - 2)
        hn = h.numpy()
        total = sum(float(log_softmax64(process(tf[r, t][None], hn[None], t, None, rp, nr), temperature)[0, hn[t + 1]])
                    for t in range(nsc))
        assert abs(total - sc) <= 1e-9 * max(1.0, abs(sc)), (r, total, sc)
    print(f"[repetition] beam n{nr} penalty {rp}: {seen['steps']} steps, {len(seen['diverged'])} latents set aside, "
          f"lengths {[len(b[0][0]) for b in out]}")


def test_graph_replay_equals_eager(full):
    m, _ = full
    z = latents(3, 8).to(DEV)
    kw = dict(temperature=0.7, top_k=40, top_p=0.9, repetition_penalty=1.3, no_repeat_ngram_size=2)
    res = []
    for graph in (False, True, True):          # the second graphed run replays the captured chunk from its first chunk on
        torch.manual_seed(99)
        res.append(m.decode_ids(z, return_logits=True, graph=graph, **kw))
    for rows, rec in res[1:]:
        assert all(torch.equal(a, b) for a, b in zip(res[0][0], rows)) and torch.equal(res[0][1], rec)
    beams = [m.decode_beams(z, 4, graph=graph, repetition_penalty=1.2, no_repeat_ngram_size=3) for graph in (False, True, True)]
    assert _same_beams(beams[0], beams[1]) and _same_beams(beams[0], beams[2])


def test_i2t_with_repetition_knobs_through_the_public_surface(tmp_path, monkeypatch):
    monkeypatch.setenv("VDB_TEXT_FLOWS", "1")
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
    from lib.model_zoo.ddim import DDIMSampler
    from oracle import weights
    from oracle.make_golden import MINI_UNET, WEIGHT_SEED
    cfg = model_cfg_bank()('vd_four_flow_v1-0')
    cfg.args.ctx_cfg_list = []
    cfg.args.vae_cfg_list = [v for v in cfg.args.vae_cfg_list if v[0] == "text"]
    cfg.args.vae_cfg_list[0][1].args.decoder.args.config.n_layer = 2
    for _, d in cfg.args.diffuser_cfg_list:
        d.args.update(MINI_UNET)
    net = get_model()(cfg, verbose=False)
    sd = weights.synth_state_dict(weights.param_shapes(net), seed=WEIGHT_SEED)
    assert not net.load_state_dict(sd, strict=False).unexpected_keys
    net.eval()
    net.to(DEV)
    g = torch.Generator().manual_seed(41)
    xT = torch.randn(2, 768, generator=g)
    c, u = torch.randn(2, 257, 768, generator=g) * 0.5, torch.zeros(2, 257, 768)
    with torch.no_grad():
        x, _ = DDIMSampler(net).sample(
            steps=4, shape=[2, 768], x_info={"type": "text", "xt": xT.clone()},
            c_info={"type": "image", "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                    "unconditional_guidance_scale": 7.5}, verbose=False, eta=0.)
    monkeypatch.chdir(tmp_path)
    vocab_dir = tmp_path / "lib" / "model_zoo" / "optimus_models" / "vocab"
    vocab_dir.mkdir(parents=True)
    (vocab_dir / "gpt2-vocab.json").write_text(json.dumps({("Ġw%d" % i): i for i in range(50257)}), encoding="utf-8")
    kw = dict(repetition_penalty=1.2, no_repeat_ngram_size=3)
    torch.manual_seed(5)
    texts = net.vae_decode(x, which='text', **kw)
    assert isinstance(texts, list) and len(texts) == 2 and all(isinstance(t, str) for t in texts)
    torch.manual_seed(5)
    assert net.vae_decode(x, which='text', **kw) == texts
    beams = net.vae_decode(x, which='text', num_beams=4, **kw)
    assert isinstance(beams, list) and len(beams) == 2 and all(isinstance(t, str) for t in beams)
    with pytest.raises(ValueError, match="no_repeat_ngram_size"):
        net.vae_decode(x, which='text', no_repeat_ngram_size=-1)
    print("[repetition] i2t texts:", texts, "beam texts:", beams)
