"""Top-k / nucleus cuts of the text sampler on the GPU (vdb_textdec_sample_filtered): picks against the fp64 oracle
(oracle/text_filter_oracle.py) over the fixture's grid, the exact kept set and the Philox distribution on a small vocabulary,
greedy decoding, bitwise equality with vdb_textdec_sample when the cuts are off, a full-size filtered decode checked step by step,
and net.vae_decode(x, 'text', top_p=...) through the public surface.

Exemption at the nucleus boundary: the kernel sums fixed-point masses exactly, the oracle in fp64.  A pick that differs from the
oracle's is excused (counted and printed) when it is the oracle's pick with top_p moved by 1e-5 either way, or when u lies within
1e-6 of a step of the oracle's CDF (the kernel's fp32 exp against the oracle's fp64 exp)."""
import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
V = 50260
NEAR = 1e-5


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _sample(logits, temperature=1.0, top_k=0, top_p=0.0, uniforms=None, seed=None, steps=1, entry="ops"):
    """Token s+1 of every row for s < steps -> int64 [R, steps].  entry: 'ops' (ops.textdec_sample), or 'filtered' / 'plain' for
    the C entry points vdb_textdec_sample_filtered / vdb_textdec_sample called directly."""
    from vdb200 import ops
    from vdb200._lib import lib, check
    R, Vr = logits.shape
    dl = logits.to(DEV).contiguous()
    tokens = torch.zeros(R, 33, dtype=torch.int32, device=DEV)
    out = []
    for s in range(steps):
        done, lengths = torch.zeros(R, dtype=torch.int32, device=DEV), torch.zeros(R, dtype=torch.int32, device=DEV)
        step = torch.tensor([s], dtype=torch.int32, device=DEV)
        if entry == "ops":
            ops.textdec_sample(dl, tokens, done, lengths, step, temperature=temperature, uniforms=uniforms, seed=seed, eos=-1,
                               max_len=1 << 30, top_k=top_k, top_p=top_p)
        else:
            tail = (_ptr(seed), _ptr(uniforms), uniforms.stride(0) if uniforms is not None else 0, None, 0, _ptr(tokens), 33,
                    _ptr(done), _ptr(lengths), _ptr(step), -1, 1 << 30, None, None)
            if entry == "filtered":
                check(lib.vdb_textdec_sample_filtered(_ptr(dl), R, Vr, Vr, float(temperature), int(top_k), float(top_p), *tail))
            else:
                check(lib.vdb_textdec_sample(_ptr(dl), R, Vr, Vr, float(temperature), *tail))
        out.append(tokens[:, s + 1].clone())
    return torch.stack(out, 1).cpu().long()


def _check_picks(got, l, top_k, top_p, u, what):
    """Asserts the kernel's picks got [n] of one row (scaled logits l, uniforms u [n]) against the oracle's -> number excused."""
    from oracle.text_filter_oracle import filter_keep_mask, filtered_pick
    want, dist = filtered_pick(l, filter_keep_mask(l, top_k, top_p), u)
    excused = (got != want) & (dist < 1e-6)
    if 0.0 < top_p < 1.0:
        lo, _ = filtered_pick(l, filter_keep_mask(l, top_k, top_p - NEAR), u)
        hi, _ = filtered_pick(l, filter_keep_mask(l, top_k, min(top_p + NEAR, 1.0 - 1e-9)), u)
        excused |= (got != want) & ((got == lo) | (got == hi))
    bad = (got != want) & ~excused
    assert not bad.any(), (what, bad.nonzero().flatten()[:4], got[bad][:4], want[bad][:4])
    return int(excused.sum())


def test_picks_match_the_oracle_on_the_grid():
    """16 rows (the fixture's seven, tie rows included, then nine seeded) x 32 given uniforms (u = 0 and 1 - 1e-12 among them)
    for every (top_k, top_p, temperature) of the fixture's grid."""
    from oracle.make_text_filter_golden import TEMPERATURE, TOP_K, TOP_P, filter_rows
    from oracle.text_filter_oracle import scaled_logits
    g = torch.Generator().manual_seed(31)
    logits = torch.cat([filter_rows(), torch.randn(9, V, generator=g) * 3])
    u = torch.rand(16, 32, generator=g, dtype=torch.float64)
    u[:, 0], u[:, 1] = 0.0, 1.0 - 1e-12
    ud = u.to(DEV)
    picks = exempt = 0
    for temp in TEMPERATURE:
        ls = [scaled_logits(logits[r], temp) for r in range(16)]
        for k in TOP_K:
            for p in TOP_P:
                got = _sample(logits, temp, k, p, uniforms=ud, steps=32)
                for r in range(16):
                    exempt += _check_picks(got[r], ls[r], k, p, u[r], (temp, k, p, r))
                    picks += got.shape[1]
    print(f"[textfilter] grid picks: {picks - exempt} of {picks} equal to the oracle, {exempt} exempt")
    assert exempt < picks // 100


def test_small_vocabulary_kept_set_and_philox_distribution():
    """V = 32: a sweep of 4096 uniforms reaches exactly the oracle's kept set; 2^16 Philox draws (16 rows x 32 steps x 128 seeds)
    against the filtered distribution give a chi-square p > 1e-3."""
    from scipy.stats import chisquare
    from oracle.text_filter_oracle import filter_keep_mask, scaled_logits
    Vs = 32
    lg = torch.linspace(-2.0, 2.0, Vs)[torch.randperm(Vs, generator=torch.Generator().manual_seed(2))].repeat(16, 1)
    seed = lambda v: torch.tensor([v], dtype=torch.int64, device=DEV)
    for temp, k, p in ((1.0, 5, 0.0), (1.0, 0, 0.6), (0.7, 8, 0.7), (1.3, 20, 0.9)):
        keep = filter_keep_mask(scaled_logits(lg[0], temp), k, p)
        u = ((torch.arange(16 * 32 * 8, dtype=torch.float64) + 0.5) / (16 * 32 * 8)).view(8, 16, 32)
        seen = torch.cat([_sample(lg, temp, k, p, uniforms=u[c].to(DEV), steps=32).flatten() for c in range(8)])
        assert set(seen.tolist()) == set(keep.nonzero().flatten().tolist()), (temp, k, p)
        counts = torch.zeros(Vs, dtype=torch.float64)
        for j in range(128):
            counts += torch.bincount(_sample(lg, temp, k, p, seed=seed(1000 + 7919 * j), steps=32).flatten(), minlength=Vs).double()
        q = torch.where(keep, torch.softmax(scaled_logits(lg[0], temp).double(), -1), torch.zeros(Vs, dtype=torch.float64))
        q = q / q.sum()
        assert counts[~keep].sum() == 0
        stat, pval = chisquare(counts[keep].numpy(), (q[keep] * counts.sum()).numpy())
        print(f"[textfilter] V=32 T={temp} top_k={k} top_p={p}: {int(keep.sum())} kept, chi-square {stat:.2f}, p {pval:.4f}")
        assert counts.sum() == 1 << 16 and pval > 1e-3


def test_greedy_is_the_argmax():
    g = torch.Generator().manual_seed(12)
    logits = torch.randn(16, V, generator=g) * 3
    assert (logits.topk(2, -1).values[:, 0] > logits.topk(2, -1).values[:, 1]).all()
    u = torch.rand(16, 32, generator=g, dtype=torch.float64)
    u[:, 0], u[:, 1] = 0.0, 1.0 - 1e-12
    want = logits.argmax(-1)[:, None].expand(16, 32)
    for temp in (0.7, 1.0, 1.3):
        assert torch.equal(_sample(logits, temp, 1, 0.0, uniforms=u.to(DEV), steps=32), want)
        assert torch.equal(_sample(logits, temp, 1, 0.9, seed=torch.tensor([77], dtype=torch.int64, device=DEV), steps=8),
                           want[:, :8])


def test_cuts_off_are_bitwise_the_plain_sampler():
    g = torch.Generator().manual_seed(13)
    logits = torch.randn(16, V, generator=g) * 3
    u = torch.rand(16, 32, generator=g, dtype=torch.float64).to(DEV)
    seed = torch.tensor([4321], dtype=torch.int64, device=DEV)
    for temp in (0.7, 1.0):
        plain_u = _sample(logits, temp, uniforms=u, steps=32, entry="plain")
        plain_s = _sample(logits, temp, seed=seed, steps=32, entry="plain")
        for k, p in ((0, 0.0), (0, 1.0), (V, 0.0), (60000, 1.0)):
            assert torch.equal(_sample(logits, temp, k, p, uniforms=u, steps=32, entry="filtered"), plain_u), (temp, k, p)
            assert torch.equal(_sample(logits, temp, k, p, seed=seed, steps=32, entry="filtered"), plain_s), (temp, k, p)


@pytest.fixture(scope="module")
def full():
    from test_text_decode_gpu import build_decoder
    return build_decoder(12, seed=11)


def test_full_size_decode_with_cuts(full):
    """top_k=40, top_p=0.9, T=0.7: every drawn token is in the oracle's kept set of the recorded logits, the recorded logits
    follow the fp32 oracle, the same seed repeats bitwise and graph replay equals eager."""
    from oracle.text_dec_oracle import gpt2_latent_logits
    from oracle.text_filter_oracle import filter_keep_mask, scaled_logits
    from test_text_decode_gpu import cmp_positions
    m, sd = full
    kw = dict(temperature=0.7, top_k=40, top_p=0.9)
    z = torch.randn(4, 768, generator=torch.Generator().manual_seed(17)) * 3.0
    torch.manual_seed(123)
    rows, rec = m.decode_ids(z.to(DEV), return_logits=True, **kw)
    exempt = 0
    for r, row in enumerate(rows):
        assert row[0] == 50258 and row[-1] == 50259 and len(row) <= 30, row
        n = min(len(row) - 1, rec.shape[0])
        for s in range(n):
            l = scaled_logits(rec[s, r].cpu(), 0.7)
            tok = int(row[s + 1])
            if not bool(filter_keep_mask(l, 40, 0.9)[tok]):
                assert bool(filter_keep_mask(l, 40, 0.9 + NEAR)[tok]), (r, s, tok)
                exempt += 1
        ref = gpt2_latent_logits(sd, z[r:r + 1], row[None, :n])[0]
        cmp_positions(rec[:n, r], ref, f"top_k 40 top_p 0.9 row {r} ({len(row)} tokens) per-step logits vs oracle")
    print(f"[textfilter] full-size decode: {sum(min(len(r) - 1, rec.shape[0]) for r in rows)} draws in the kept set, {exempt} exempt")
    torch.manual_seed(123)
    again, rec2 = m.decode_ids(z.to(DEV), return_logits=True, **kw)
    assert all(torch.equal(a, b) for a, b in zip(rows, again)) and torch.equal(rec, rec2)
    res = []
    for graph in (False, True, True):
        torch.manual_seed(99)
        res.append(m.decode_ids(z.to(DEV), return_logits=True, graph=graph, **kw))
    for rr, rc in res[1:]:
        assert all(torch.equal(a, b) for a, b in zip(res[0][0], rr)) and torch.equal(res[0][1], rc)


def test_vae_decode_top_p_through_the_public_surface(tmp_path, monkeypatch):
    monkeypatch.setenv("VDB_TEXT_FLOWS", "1")
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
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
    x = torch.randn(3, 768, generator=torch.Generator().manual_seed(41)).to(DEV)
    monkeypatch.chdir(tmp_path)
    vocab_dir = tmp_path / "lib" / "model_zoo" / "optimus_models" / "vocab"
    vocab_dir.mkdir(parents=True)
    (vocab_dir / "gpt2-vocab.json").write_text(json.dumps({("Ġw%d" % i): i for i in range(50257)}), encoding="utf-8")
    torch.manual_seed(5)
    texts = net.vae_decode(x, which='text', top_p=0.9)
    assert isinstance(texts, list) and len(texts) == 3 and all(isinstance(t, str) for t in texts)
    torch.manual_seed(5)
    assert net.vae_decode(x, which='text', top_p=0.9) == texts
    torch.manual_seed(5)
    greedy = net.vae_decode(x, which='text', top_k=1)
    torch.manual_seed(6)
    assert net.vae_decode(x, which='text', top_k=1) == greedy          # greedy does not depend on the draws
    with pytest.raises(ValueError, match="top_p"):
        net.vae_decode(x, which='text', top_p=1.5)
    print("[textfilter] top_p 0.9 texts:", texts)
