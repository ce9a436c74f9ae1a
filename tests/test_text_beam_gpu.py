"""Text decoder beam search on the GPU: vdb_textdec_beam_step against the fp64 oracle (oracle/text_beam_oracle.py) on a grid of
row layouts, vocabularies, temperatures, steps, finished beams, exact ties and -1e30 logits; the KV-cache attention through a
src table against the plain one on a physically gathered cache; a full-size decode replayed step by step through the oracle on its own
recorded logits; returned scores re-scored from teacher-forced and fp64-oracle logits; width 1 against greedy decoding; graph
replay, repeatability and the group split; and net.vae_decode(x, 'text', num_beams=4).

Exemption: a selection whose fp64 margin in the oracle (the smallest relative gap between consecutive candidates among a
latent's K + 1 best that are not exact ties) is below 1e-12 may legitimately go either way; such latents are counted and printed,
not compared.  Exact ties are compared: both sides compute them from identical values."""
import json

import numpy as np
import pytest
import torch

from lib.model_zoo.optimus import decode_plan
from oracle.text_beam_oracle import BeamState, beam_step, log_softmax64, place, rank_final

pytestmark = pytest.mark.gpu

DEV = "cuda"
EOS, BOS = 50259, 50258
MAX_LEN = 30
NEAR = 1e-12


def _dev(a, dt):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dt).to(DEV)


def run_kernel_step(st, logits, K, s, temperature, eos=EOS, max_len=MAX_LEN):
    """vdb_textdec_beam_step on a copy of the oracle state st -> (BeamState, trace [R, 3], recorded logits [R, V])"""
    from vdb200 import ops
    R, V = logits.shape
    tokens, src = _dev(st.tokens, torch.int32), _dev(st.src, torch.int32)
    scores, done, lengths = _dev(st.scores, torch.float64), _dev(st.done, torch.int32), _dev(st.lengths, torch.int32)
    step = torch.tensor([s], dtype=torch.int32, device=DEV)
    cand_tok = torch.full((R * K,), -7, dtype=torch.int32, device=DEV)
    cand_logp = torch.zeros(R * K, dtype=torch.float64, device=DEV)
    record = torch.full((s + 1, R, V), float("nan"), device=DEV)
    trace = torch.full((s + 1, R, 3), float("nan"), dtype=torch.float64, device=DEV)
    ops.textdec_beam_step(_dev(logits, torch.float32), K, tokens, src, scores, done, lengths, step, cand_tok, cand_logp,
                          temperature=temperature, eos=eos, max_len=max_len, record=record, trace=trace)
    new = BeamState(tokens.cpu().long().numpy(), src.cpu().long().numpy(), scores.cpu().numpy(), done.cpu().numpy() != 0,
                    lengths.cpu().long().numpy())
    return new, trace[s].cpu().numpy(), record[s].cpu().numpy()


def compare_step(got, gtrace, want, wtrace, margins, K, what):
    """exact equality of everything but scores (1e-12 relative) per latent; -> latents exempted as near-ties"""
    exempt = 0
    for i, mg in enumerate(margins):
        rows = slice(i * K, (i + 1) * K)
        if mg < NEAR:
            exempt += 1
            print(f"[beam] {what}: latent {i} exempt, oracle margin {mg:.3g}")
            continue
        assert np.array_equal(gtrace[rows, :2], wtrace[rows, :2]), (what, i, gtrace[rows, :2], wtrace[rows, :2])
        for name in ("tokens", "src", "done", "lengths"):
            assert np.array_equal(getattr(got, name)[rows], getattr(want, name)[rows]), (what, i, name)
        a, b = got.scores[rows], want.scores[rows]
        same = (a == b) | (np.abs(a - b) <= NEAR * np.maximum(np.abs(b), 1.0))
        assert same.all(), (what, i, a, b)
        assert np.array_equal(gtrace[rows, 2], a)
    return exempt


def grid_case(n, K, V, s, seed):
    """(oracle state before step s, fp32 logits [n K, V]) with finished beams, exact ties across tokens and beams, -1e30 logits"""
    rng = np.random.default_rng(seed)
    R = n * K
    st = BeamState.start(n, K, BOS, EOS)
    logits = (rng.standard_normal((R, V)) * 3).astype(np.float32)
    logits[:, rng.integers(0, V, 3)] = logits[:, [0]]                       # duplicated values across tokens
    top = logits.argmax(1)
    logits[np.arange(R), (top + 5) % V] = logits[np.arange(R), top]         # a tie for the maximum
    logits[:, rng.integers(0, V, V // 4)] = -1e30
    if s > 0:
        st.tokens[:, 1:s + 1] = rng.integers(0, V, (R, s))
        st.src[:, :s] = rng.integers(0, R, (R, s))
        st.scores[:] = -np.sort(rng.uniform(0.5, 40.0, R))
        for r in range(R):
            if rng.random() < 0.3:                                             # finished earlier with a chosen <eos>
                L = int(rng.integers(2, s + 2))
                st.done[r], st.lengths[r] = True, L
                st.tokens[r, L - 1] = EOS
        for i in range(n):                                                     # two live beams of one latent exactly tied
            b = i * K
            if K >= 2 and not st.done[b] and not st.done[b + 1]:
                st.scores[b + 1] = st.scores[b]
                logits[b + 1] = logits[b]
    return st, logits


@pytest.mark.parametrize("s", [0, 13, MAX_LEN - 3])
@pytest.mark.parametrize("temperature", [1.0, 0.7])
@pytest.mark.parametrize("V", [40, 50260])
@pytest.mark.parametrize("n,K", [(1, 1), (16, 1), (4, 4), (3, 5), (2, 8), (1, 16)])
def test_beam_step_matches_oracle(n, K, V, temperature, s):
    st, logits = grid_case(n, K, V, s, seed=1000 * n + 37 * K + V + s)
    got, gtrace, rec = run_kernel_step(st, logits, K, s, temperature)
    want, wtrace, margins = beam_step(st, logits, K, s, EOS, MAX_LEN, temperature)
    assert np.array_equal(rec, logits), "record must hold this step's logits per physical row"
    exempt = compare_step(got, gtrace, want, wtrace, margins, K, f"n{n} K{K} V{V} T{temperature} s{s}")
    print(f"[beam] grid n{n} K{K} V{V} T{temperature} s{s}: {n - exempt} latents equal, {exempt} near-tie exemptions")
    if s == MAX_LEN - 3:                                                       # every beam finishes at the last step
        assert got.done.all()
    again, atrace, _ = run_kernel_step(st, logits, K, s, temperature)
    assert np.array_equal(again.scores, got.scores) and np.array_equal(atrace, gtrace), "must repeat bitwise"


@pytest.mark.parametrize("s", [0, 1, 17, 30, 31])
def test_attention_src_equals_attention_on_a_gathered_cache(s):
    from vdb200 import ops
    R, H, T = 16, 12, 32
    D = H * 64
    g = torch.Generator().manual_seed(s)
    qkv = torch.randn(R, 3 * D, generator=g).to(DEV)
    mem = torch.randn(R, D, generator=g).to(DEV)
    kc, vc = torch.randn(R, H, T, 64, generator=g).to(DEV), torch.randn(R, H, T, 64, generator=g).to(DEV)
    step = torch.tensor([s], dtype=torch.int32, device=DEV)
    tables = {"identity": torch.arange(R)[:, None].expand(R, T), "one parent": torch.full((R, T), 5),
              "reversed": (R - 1 - torch.arange(R))[:, None].expand(R, T), "random": torch.randint(0, R, (R, T), generator=g)}
    for name, src in tables.items():
        src = src.to(torch.int32).contiguous().to(DEV)
        k1, v1, o1 = kc.clone(), vc.clone(), torch.empty(R, D, device=DEV)
        ops.textdec_attention(qkv, mem, k1, v1, step, o1, src=src)
        idx = src.long()[:, None, :, None].expand(R, H, T, 64)
        kg, vg = torch.gather(kc, 0, idx).contiguous(), torch.gather(vc, 0, idx).contiguous()
        o2 = torch.empty(R, D, device=DEV)
        ops.textdec_attention(qkv, mem, kg, vg, step, o2)
        assert torch.equal(o1, o2), (name, s)
        want_k, want_v = kc.clone(), vc.clone()
        want_k[:, :, s] = qkv[:, D:2 * D].reshape(R, H, 64)
        want_v[:, :, s] = qkv[:, 2 * D:].reshape(R, H, 64)
        assert torch.equal(k1, want_k) and torch.equal(v1, want_v), (name, s)


@pytest.fixture(scope="module")
def full():
    from test_text_decode_gpu import build_decoder
    return build_decoder(12, seed=11)


def latents(n, seed):
    return torch.randn(n, 768, generator=torch.Generator().manual_seed(seed)) * 3.0


@pytest.mark.parametrize("temperature", [1.0, 0.7])
def test_full_beam_plan_decode_follows_the_oracle_step_by_step(full, temperature):
    m, _ = full
    n, K = 4, 4
    z = latents(n, 21)
    out, st, ran = m._beam_group(z.to(DEV), decode_plan("beam", temperature, EOS, record=True, num_beams=K), 1.0, 1.0)
    rec, trace = st.record[:ran].cpu().numpy(), st.trace[:ran].cpu().numpy()
    ost = BeamState.start(n, K, BOS, EOS)
    exempt = 0
    for s in range(ran):
        new, wtrace, margins = beam_step(ost, rec[s], K, s, EOS, MAX_LEN, temperature)
        for i in range(n):
            rows = slice(i * K, (i + 1) * K)
            if margins[i] < NEAR:
                # a near-tie may go either way: adopt the kernel's selection for this latent and keep replaying
                exempt += 1
                print(f"[beam] full decode T{temperature}: step {s} latent {i} exempt, oracle margin {margins[i]:.3g}")
                for j in range(K):
                    p, v, sc = trace[s, i * K + j]
                    place(new, ost, i * K + j, i * K + int(p), int(v), sc, s, EOS, MAX_LEN)
                continue
            assert np.array_equal(trace[s, rows, :2], wtrace[rows, :2]), (s, i, trace[s, rows], wtrace[rows])
            a, b = trace[s, rows, 2], wtrace[rows, 2]
            assert ((a == b) | (np.abs(a - b) <= NEAR * np.abs(b))).all(), (s, i, a, b)
        ost = new
    print(f"[beam] full decode T{temperature}: {ran} steps, {exempt} near-tie exemptions, lengths {[len(b[0][0]) for b in out]}")
    assert ost.done.all()
    want = rank_final(ost, K, MAX_LEN)
    for i in range(n):
        for (ids, sc, nm), (wids, wsc, wnm) in zip(out[i], want[i]):
            assert ids.tolist() == wids.tolist() and abs(sc - wsc) <= NEAR * abs(wsc)


def test_returned_scores_rescore_from_teacher_forced_and_oracle_logits(full):
    from oracle.text_dec_oracle import gpt2_latent_logits
    from test_text_decode_gpu import TOL
    m, sd = full
    n, K, temperature = 4, 4, 0.7
    z = latents(n, 22)
    out = m.decode_beams(z.to(DEV), K, temperature=temperature)
    hyps = [(i, ids, sc) for i in range(n) for ids, sc, _ in out[i]]
    L = max(len(ids) for _, ids, _ in hyps)
    ids = torch.full((len(hyps), L), EOS, dtype=torch.long)
    for r, (_, h, _) in enumerate(hyps):
        ids[r, :len(h)] = h
    zr = z[[i for i, _, _ in hyps]]
    tf = m.teacher_forced_logits(zr.to(DEV), ids).cpu()
    ref = gpt2_latent_logits(sd, zr, ids)
    for r, (_, h, sc) in enumerate(hyps):
        nsc = min(len(h) - 1, MAX_LEN - 2)
        lp_tf = log_softmax64(tf[r, :nsc].numpy(), temperature)
        lp_ref = log_softmax64(ref[r, :nsc].numpy(), temperature)
        tgt = h[1:nsc + 1].numpy()
        s_tf = lp_tf[np.arange(nsc), tgt].sum()
        s_ref = lp_ref[np.arange(nsc), tgt].sum()
        assert abs(s_tf - sc) <= 1e-6 * max(1.0, abs(sc)), (r, s_tf, sc)
        bound = sum(2 * TOL * float(ref[r, t].abs().max()) / temperature for t in range(nsc))
        assert abs(s_ref - sc) <= bound, (r, s_ref, sc, bound)
    print(f"[beam] re-scored {len(hyps)} hypotheses from teacher-forced and fp64-oracle logits")


def test_width_one_is_greedy_decoding(full):
    """equal token for token (top_k=1 would draw among exactly tied maxima; random weights give none)"""
    m, _ = full
    z = latents(4, 23).to(DEV)
    beam = m.decode_ids(z, num_beams=1)
    greedy = m.decode_ids(z, top_k=1)
    assert all(torch.equal(a, b) for a, b in zip(beam, greedy)), (beam, greedy)


def _same(a, b):
    return all(len(x) == len(y) and all(torch.equal(p[0], q[0]) and p[1] == q[1] and p[2] == q[2] for p, q in zip(x, y))
               for x, y in zip(a, b)) and len(a) == len(b)


def test_graph_replay_repeatability_and_groups(full):
    m, _ = full
    z = latents(6, 24).to(DEV)
    torch.manual_seed(1)
    eager = m.decode_beams(z[:4], 4, graph=False)
    torch.manual_seed(2)
    first = m.decode_beams(z[:4], 4)
    torch.manual_seed(3)
    second = m.decode_beams(z[:4], 4)
    assert _same(eager, first) and _same(first, second), "graph replay must equal eager, and calls must repeat"
    split = m.decode_beams(z, 4)                                     # 6 x 4 rows: groups of 4 and 2 latents
    assert len(split) == 6 and _same(split, first + m.decode_beams(z[4:], 4))
    assert [b[0][0].tolist() for b in split] == [r.tolist() for r in m.decode_ids(z, num_beams=4)]


def test_i2t_beam_search_through_the_public_surface(tmp_path, monkeypatch):
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
    texts = net.vae_decode(x, which='text', num_beams=4)
    assert isinstance(texts, list) and len(texts) == 2 and all(isinstance(t, str) for t in texts)
    assert net.vae_decode(x, which='text', num_beams=4) == texts
    with pytest.raises(ValueError):
        net.vae_decode(x, which='text', num_beams=4, top_k=5)
    print("[beam] i2t beam texts:", texts)
