"""Optimus text decoder on the GPU: teacher-forced logits against the reference's golden and the fp32 oracle, sampled decodes
checked step by step against the oracle, the sampler's inverse CDF and Philox stream, graph replay against eager launches, and
i2t end to end through DDIMSampler and VD_v2_0.vae_decode.

Tolerance of the logits: weights and the GEMV operands (LayerNorm outputs, attention / MLP activations) are rounded to bf16
(relative error <= 2^-9 each) with fp32 accumulation.  Over 768- to 3072-term dot products of random-sign terms these errors
average out to well under 1% of the largest logit of a position; 2% (cosine >= 0.999) leaves room for 12 layers of that."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"
TOL = 2e-2
EOS, BOS = 50259, 50258


def build_decoder(n_layer, seed=7):
    from lib.model_zoo.optimus import optimus_vae_next
    from oracle.make_text_golden import synth_decoder_state
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=n_layer)))
    sd = synth_decoder_state({k: tuple(v.shape) for k, v in m.state_dict().items()}) if seed == 7 else None
    if sd is None:
        from oracle import weights
        sd = {k: weights.tensor_for(k, tuple(v.shape), seed) for k, v in m.state_dict().items()
              if not k.endswith((".attn.bias", "lm_head.weight"))}
    res = m.load_state_dict(sd, strict=False)
    assert all(k.endswith((".attn.bias", "lm_head.weight")) for k in res.missing_keys), res.missing_keys
    m.to(DEV)
    sd = dict(sd)
    sd["decoder.lm_head.weight"] = sd["decoder.transformer.wte.weight"]
    return m, sd


@pytest.fixture(scope="module")
def full():
    return build_decoder(12, seed=11)


def cmp_positions(out, ref, what):
    """cosine >= 0.999 and max|err| <= TOL * max|ref| at every position ([..., V] rows)."""
    out, ref = out.float().cpu().reshape(-1, out.shape[-1]), ref.float().cpu().reshape(-1, ref.shape[-1])
    assert torch.isfinite(out).all(), what
    cos = F.cosine_similarity(out, ref, dim=-1)
    rel = (out - ref).abs().amax(-1) / ref.abs().amax(-1)
    print(f"[textdec] {what}: min cos {cos.min().item():.6f}, worst max|err|/max|ref| {rel.max().item():.4g}")
    assert cos.min().item() >= 0.999 and rel.max().item() <= TOL, what


def test_module_keys_and_tied_head_on_gpu():
    keys = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLD, "keys_text_dec.json"))).items()}
    m, _ = build_decoder(2)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == keys
    assert m.decoder.lm_head.weight.data_ptr() == m.decoder.transformer.wte.weight.data_ptr()


def test_teacher_forced_logits_vs_reference_golden():
    from test_text_decode import check_against_golden
    gold = dict(np.load(os.path.join(GOLD, "text_dec.npz")))
    m, _ = build_decoder(int(gold["n_layer"]))
    logits = m.teacher_forced_logits(torch.from_numpy(gold["z"]).to(DEV), torch.from_numpy(gold["ids"]))
    worst = check_against_golden(logits, gold, rel=TOL)
    print(f"[textdec] 2-layer teacher-forced logits vs reference golden: worst {worst:.4g} of max|logit|")


def test_teacher_forced_logits_vs_oracle_full_size(full):
    from oracle.text_dec_oracle import gpt2_latent_logits
    m, sd = full
    g = torch.Generator().manual_seed(3)
    z = torch.randn(4, 768, generator=g)
    ids = torch.randint(0, 50260, (4, 20), generator=g)
    ids[:, 0] = BOS
    out = m.teacher_forced_logits(z.to(DEV), ids)
    ref = gpt2_latent_logits(sd, z, ids)
    cmp_positions(out, ref, "12-layer teacher-forced logits vs oracle")
    assert torch.equal(out, m.teacher_forced_logits(z.to(DEV), ids, graph=True)), "graph replay must equal eager"


@pytest.mark.parametrize("temperature", [1.0, 0.7])
def test_sampled_decode_follows_the_oracle_step_by_step(full, temperature):
    from oracle.text_dec_oracle import gpt2_latent_logits
    m, sd = full
    g = torch.Generator().manual_seed(17)
    z = torch.randn(4, 768, generator=g) * 3.0      # latents of the diffusion's scale
    torch.manual_seed(123)
    rows, rec = m.decode_ids(z.to(DEV), temperature=temperature, return_logits=True)
    assert len(rows) == 4
    for r, row in enumerate(rows):
        assert row[0] == BOS and row[-1] == EOS and len(row) <= 30, row
        assert (row[1:-1] != EOS).all()
        n = min(len(row) - 1, rec.shape[0])                                    # a forced final <EOS> had no draw
        ref = gpt2_latent_logits(sd, z[r:r + 1], row[None, :n])[0]             # the oracle on the product's own tokens
        cmp_positions(rec[:n, r], ref, f"T={temperature} row {r} ({len(row)} tokens) per-step logits vs oracle")
    # the same seed gives the same tokens; an eos_token the first run drew at step 3 ends that row there, frozen afterwards
    torch.manual_seed(123)
    assert all(torch.equal(a, b) for a, b in zip(rows, m.decode_ids(z.to(DEV), temperature=temperature)))
    r = next(i for i, row in enumerate(rows) if len(row) > 5)
    stop = int(rows[r][3])
    torch.manual_seed(123)
    again = m.decode_ids(z.to(DEV), temperature=temperature, eos_token=stop)
    cut = next(j for j in range(1, len(rows[r])) if int(rows[r][j]) == stop)
    assert torch.equal(again[r], rows[r][:cut + 1]), (again[r], rows[r])


def _sampler_inputs(R, V, seed):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(R, V, generator=g) * 3
    return logits


def _run_sampler(logits, temperature=1.0, uniforms=None, seed=None, steps=1):
    from vdb200 import ops
    R = logits.shape[0]
    dl = logits.to(DEV)
    tokens = torch.zeros(R, 33, dtype=torch.int32, device=DEV)
    out = []
    for s in range(steps):
        done, lengths = torch.zeros(R, dtype=torch.int32, device=DEV), torch.zeros(R, dtype=torch.int32, device=DEV)
        step = torch.tensor([s], dtype=torch.int32, device=DEV)
        ops.textdec_sample(dl, tokens, done, lengths, step, temperature=temperature, uniforms=uniforms, seed=seed, eos=-1,
                           max_len=1 << 30)
        out.append(tokens[:, s + 1].clone())
    return torch.stack(out, 1).cpu()


def test_sampler_inverse_cdf_matches_fp64():
    R, V = 16, 50260
    for temperature in (1.0, 0.7):
        logits = _sampler_inputs(R, V, 5)
        g = torch.Generator().manual_seed(9)
        u = torch.rand(R, 32, generator=g, dtype=torch.float64)
        u[0, :4] = torch.tensor([0.0, 1e-12, 1 - 1e-12, 0.5], dtype=torch.float64)
        got = _run_sampler(logits, temperature, uniforms=u.to(DEV), steps=32)
        p = torch.softmax(logits.double() / temperature, -1)
        cdf = p.cumsum(-1)
        cdf = cdf / cdf[:, -1:]
        want = torch.searchsorted(cdf, u, right=True).clamp_max(V - 1)
        near = torch.zeros_like(want, dtype=torch.bool)
        for r in range(R):
            d = (cdf[r][None, :] - u[r][:, None]).abs().amin(-1)
            near[r] = d < 1e-6
        mism = (got != want) & ~near
        assert not mism.any(), (temperature, mism.nonzero()[:5], got[mism][:5], want[mism][:5])


def test_sampler_philox_stream():
    logits = _sampler_inputs(4, 50260, 6)
    seed = lambda v: torch.tensor([v], dtype=torch.int64, device=DEV)
    a = _run_sampler(logits, seed=seed(1234), steps=8)
    assert torch.equal(a, _run_sampler(logits, seed=seed(1234), steps=8)), "same seed must repeat bitwise"
    assert not torch.equal(a, _run_sampler(logits, seed=seed(1235), steps=8)), "different seeds must differ"
    # chi-square over 2^16 draws (16 rows x 32 steps x 128 seeds) of a fixed 32-token distribution: deterministic, p > 1e-3
    from scipy.stats import chisquare
    V = 32
    lg = torch.linspace(-2.0, 2.0, V).repeat(16, 1)
    counts = torch.zeros(V, dtype=torch.float64)
    for k in range(128):
        draws = _run_sampler(lg, seed=seed(1000 + 7919 * k), steps=32)
        counts += torch.bincount(draws.flatten().long(), minlength=V).double()
    p = torch.softmax(lg[0].double(), -1)
    stat, pval = chisquare(counts.numpy(), (p * counts.sum()).numpy())
    print(f"[textdec] Philox chi-square over {int(counts.sum())} draws: stat {stat:.2f}, p {pval:.4f}")
    assert counts.sum() == 1 << 16 and pval > 1e-3


def test_graph_replay_equals_eager(full):
    m, _ = full
    z = torch.randn(3, 768, generator=torch.Generator().manual_seed(8)).to(DEV) * 3.0
    res = []
    for graph in (False, True, True):          # the second graphed run replays the captured chunk from its first chunk on
        torch.manual_seed(99)
        res.append(m.decode_ids(z, return_logits=True, graph=graph))
    for rows, rec in res[1:]:
        assert all(torch.equal(a, b) for a, b in zip(res[0][0], rows))
        assert torch.equal(res[0][1], rec)


def test_i2t_through_the_public_surface(tmp_path, monkeypatch):
    """DDIMSampler.sample on a text latent, then net.vae_decode(x, 'text') with a synthetic vocabulary at the default path."""
    monkeypatch.setenv("VDB_TEXT_FLOWS", "1")
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.optimus import VocabularyMissingError
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
    with pytest.raises(VocabularyMissingError):
        net.vae_decode(x, which='text', temperature=1)
    vocab_dir = tmp_path / "lib" / "model_zoo" / "optimus_models" / "vocab"
    vocab_dir.mkdir(parents=True)
    vocab = {("Ġw%d" % i): i for i in range(50257)}
    (vocab_dir / "gpt2-vocab.json").write_text(json.dumps(vocab), encoding="utf-8")
    torch.manual_seed(5)
    texts = net.vae_decode(x, which='text', temperature=1)
    assert isinstance(texts, list) and len(texts) == 2 and all(isinstance(t, str) for t in texts)
    assert all(w.startswith("w") or w in ("<PAD>", "<BOS>") for t in texts for w in t.split()), texts
    torch.manual_seed(5)
    assert net.vae_decode(x, which='text', temperature=1) == texts
    print("[textdec] i2t texts:", texts)
