"""Optimus text encoder on the GPU: the varlen flash attention and the pooler's tanh GEMV against fp64, the encoder against the
reference's golden and the 12-layer fp32 oracle, run-to-run and batch consistency, and encode -> DDIM -> decode through the public
surface.

Tolerance of the latents: weights and every GEMM operand (the LayerNorm outputs of the residual stream, attention probabilities
and outputs, GELU outputs) are bf16 with fp32 accumulation, as in the CLIP towers and the text decoder.  The criterion is the
decoder tests': cosine >= 0.999 and max|err| <= 2% of max|ref| on every row."""
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
D, HEADS = 768, 12


# ------------------------------------------------------------------------------------------------ varlen attention
def _attn_inputs(B, Lp, H, seed, garbage=None, kv_len=None):
    """q | k bf16 [B*Lp, 2*H*64], V^T bf16 [H*64, B*Lp]; garbage: value written into the K rows / V^T columns past kv_len."""
    g = torch.Generator().manual_seed(seed)
    qk = torch.randn(B * Lp, 2 * H * 64, generator=g).to(torch.bfloat16)
    vt = torch.randn(H * 64, B * Lp, generator=g).to(torch.bfloat16)
    if garbage is not None:
        for b, n in enumerate(kv_len):
            rows = slice(b * Lp + max(n, 0), (b + 1) * Lp)
            qk[rows, H * 64:] = garbage
            vt[:, rows] = -garbage
    return qk, vt


def _attn_ref(qk, vt, B, Lp, H, kv_len):
    """fp64 softmax(q k^T / 8) v over the visible keys of each item; zero rows for an item without keys."""
    q = qk[:, :H * 64].double().view(B, Lp, H, 64).transpose(1, 2)
    k = qk[:, H * 64:].double().view(B, Lp, H, 64).transpose(1, 2)
    v = vt.double().t().reshape(B, Lp, H, 64).transpose(1, 2)
    out = torch.zeros(B, H, Lp, 64, dtype=torch.float64)
    for b, n in enumerate(kv_len):
        n = min(n, Lp)
        if n > 0:
            w = (q[b] @ k[b, :, :n].transpose(-1, -2) / 8.0).softmax(-1)
            out[b] = w @ v[b, :, :n]
    return out.transpose(1, 2).reshape(B * Lp, H * 64)


def _attn_run(qk, vt, B, Lp, H, kv_len):
    from vdb200 import ops
    out = torch.full((B * Lp, H * 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    kvl = torch.tensor(kv_len, dtype=torch.int32, device=DEV)
    ops.attention(qk.to(DEV), qk.to(DEV), vt.to(DEV), out, B, H, Lp, Lp, 64, scale=0.125, q_col0=0, k_col0=H * 64,
                  q_bstride=Lp, kv_bstride=Lp, kv_len=kvl)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("Lp, kv_len", [(80, [1, 7, 64, 77, 80]), (208, [1, 128, 129, 200])])
def test_varlen_attention_matches_fp64(Lp, kv_len):
    """every output row against fp64 on the same bf16 operands: P is rounded to bf16 before the PV product (relative error
    <= 2^-9 per weight), so each row's error stays well under 1% of max|v|"""
    B, H = len(kv_len), 4
    qk, vt = _attn_inputs(B, Lp, H, seed=Lp)
    out = _attn_run(qk, vt, B, Lp, H, kv_len)
    ref = _attn_ref(qk, vt, B, Lp, H, kv_len)
    assert torch.isfinite(out.float()).all()
    err = (out.double() - ref).abs().view(B, Lp, -1).amax(dim=(1, 2))
    scale = vt.double().abs().amax()
    print(f"[textenc] varlen attention Lp {Lp} kv_len {kv_len}: worst max|err| / max|v| {(err / scale).max().item():.3g}")
    assert (err <= 1e-2 * scale).all(), (err / scale)


def test_varlen_attention_ignores_padded_keys_and_zeroes_empty_items():
    B, Lp, H = 4, 208, 2
    kv_len = [5, 0, 130, 208]
    clean_qk, clean_vt = _attn_inputs(B, Lp, H, seed=3, garbage=0.0, kv_len=kv_len)
    dirty_qk, dirty_vt = _attn_inputs(B, Lp, H, seed=3, garbage=3.0e38, kv_len=kv_len)   # near bf16's largest finite value
    assert torch.isfinite(dirty_qk.float()).all() and torch.isfinite(dirty_vt.float()).all()
    clean = _attn_run(clean_qk, clean_vt, B, Lp, H, kv_len)
    dirty = _attn_run(dirty_qk, dirty_vt, B, Lp, H, kv_len)
    assert torch.equal(clean.view(torch.int16), dirty.view(torch.int16)), "garbage in masked K / V rows changed the output"
    assert torch.equal(clean[Lp:2 * Lp], torch.zeros(Lp, H * 64, dtype=torch.bfloat16)), "kv_len 0 must write zero rows"
    ref = _attn_ref(clean_qk, clean_vt, B, Lp, H, kv_len)
    assert (clean.double() - ref).abs().max() <= 1e-2 * clean_vt.double().abs().max()


# ------------------------------------------------------------------------------------------------ pooler GEMV
def test_tanh_gemv_matches_fp64():
    """tanh(x W^T + b) on the [CLS] rows of a token stream (row stride Lp * 768), 16 rows and a 5-row tail; x is rounded to
    bf16 in the kernel, so the reference uses the same bf16 x and W in fp64."""
    from vdb200 import ops
    g = torch.Generator().manual_seed(21)
    Lp = 24
    stream = torch.randn(21, Lp * D, generator=g) * 2.0
    w = (torch.randn(D, D, generator=g) * D ** -0.5).to(torch.bfloat16)
    b = torch.randn(D, generator=g) * 0.5
    x = stream.view(21, Lp * D)[:, :D]
    ref = torch.tanh(x.to(torch.bfloat16).double() @ w.double().t() + b.double())
    sd, wd, bd = stream.to(DEV), w.to(DEV), b.to(DEV)
    out = torch.zeros(21, D, device=DEV)
    for r0, r1 in ((0, 16), (16, 21)):
        ops.textdec_gemv(sd.view(21, Lp * D)[r0:r1, :D], wd, out[r0:r1], bias=bd, act=ops.ACT_TANH)
    err = (out.cpu().double() - ref).abs().max().item()
    print(f"[textenc] tanh GEMV max|err| {err:.3g}")
    assert err <= 2e-4
    assert (ref.abs() > 0.99).any() and (ref.abs() < 0.1).any()      # the inputs reach both the saturated and the linear range


# ------------------------------------------------------------------------------------------------ the encoder
def build_encoder(n_layer, seed=7):
    from lib.model_zoo.optimus import optimus_vae_next
    from oracle import weights
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=1)), encoder=dict(config=dict(num_hidden_layers=n_layer)))
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("encoder.")}
    sd = {k: weights.tensor_for(k, s, seed) for k, s in shapes.items()}
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and not [k for k in res.missing_keys if k.startswith("encoder.")]
    m.to(DEV)
    return m, sd


@pytest.fixture(scope="module")
def full():
    return build_encoder(12, seed=11)


def cmp_rows(out, ref, what):
    out, ref = out.float().cpu(), ref.float().cpu()
    assert torch.isfinite(out).all(), what
    cos = F.cosine_similarity(out, ref, dim=-1)
    rel = (out - ref).abs().amax(-1) / ref.abs().amax(-1)
    print(f"[textenc] {what}: min cos {cos.min().item():.6f}, worst max|err|/max|ref| {rel.max().item():.4g}")
    assert cos.min().item() >= 0.999 and rel.max().item() <= TOL, what


def _ragged_ids(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(len(lengths), max(lengths), dtype=torch.long)
    for r, n in enumerate(lengths):
        ids[r, 0], ids[r, n - 1] = 101, 102
        ids[r, 1:n - 1] = torch.randint(999, 28996, (n - 2,), generator=g)
    return ids


def test_encoder_vs_reference_golden():
    gold = dict(np.load(os.path.join(GOLD, "text_enc.npz")))
    m, _ = build_encoder(int(gold["n_layer"]), seed=int(gold["weight_seed"]))
    z = m.encode_ids(torch.from_numpy(gold["ids"]), gold["lengths"].tolist())
    assert z.shape == (6, 768) and z.dtype == torch.float32
    cmp_rows(z, torch.from_numpy(gold["z_mu"]), "2-layer z_mu vs reference golden")


@pytest.mark.parametrize("lengths", [[40], [2, 79, 13, 60], [int(v) for v in torch.randint(2, 80, (20,),
                                      generator=torch.Generator().manual_seed(4))], [202, 17, 130]],
                         ids=["n1", "n4", "n20", "max_length200"])
def test_encoder_vs_oracle_full_size(full, lengths):
    from oracle.text_enc_oracle import bert_latent_mu
    m, sd = full
    ids = _ragged_ids(lengths, seed=len(lengths))
    z = m.encode_ids(ids, lengths)
    cmp_rows(z, bert_latent_mu(sd, ids), f"12-layer z_mu vs oracle, lengths {lengths}")


def test_encoder_is_deterministic_and_batch_independent(full):
    m, _ = full
    lengths = [9, 70, 33, 79]
    ids = _ragged_ids(lengths, seed=5)
    a, b = m.encode_ids(ids, lengths), m.encode_ids(ids, lengths)
    assert torch.equal(a, b), "two calls must agree bitwise"
    alone = m.encode_ids(ids[:1, :9], [9])
    cmp_rows(alone, a[:1], "a sentence alone vs inside a batch of longer ones")


# ------------------------------------------------------------------------------------------------ the public surface
def test_encode_ddim_decode_through_the_public_surface(tmp_path, monkeypatch):
    """net.vae_encode(texts, 'text') and net.ctx_encode(texts, 'vae_text') with a synthetic vocabulary at the default path, then a
    DDIM walk from that latent (x0_forward_timesteps) and net.vae_decode(x, 'text')."""
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
    vcfg = cfg.args.vae_cfg_list[0][1].args
    vcfg.decoder.args.config.n_layer = 2
    vcfg.encoder.args.config.num_hidden_layers = 2
    for _, d in cfg.args.diffuser_cfg_list:
        d.args.update(MINI_UNET)
    net = get_model()(cfg, verbose=False)
    sd = weights.synth_state_dict(weights.param_shapes(net), seed=WEIGHT_SEED)
    assert not net.load_state_dict(sd, strict=False).unexpected_keys
    net.eval()
    net.to(DEV)
    texts = ["a red bus on a wet street.", "Two cats, asleep!", ""]
    monkeypatch.chdir(tmp_path)
    with pytest.raises(VocabularyMissingError, match="bert-base-cased-vocab.txt"):
        net.vae_encode(texts, which='text')
    vocab_dir = tmp_path / "lib" / "model_zoo" / "optimus_models" / "vocab"
    vocab_dir.mkdir(parents=True)
    words = ["a", "red", "bus", "on", "wet", "street", "two", "cat", "##s", "asleep", ".", ",", "!"]
    pieces = ["[PAD]"] + [f"[unused{i}]" for i in range(99)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    pieces += [f"w{i}" for i in range(28996 - len(pieces))]
    (vocab_dir / "bert-base-cased-vocab.txt").write_text("\n".join(pieces) + "\n", encoding="utf-8")
    z = net.vae_encode(texts, which='text')
    assert z.shape == (3, 768) and z.dtype == torch.float32 and torch.isfinite(z).all()
    assert torch.equal(z, net.ctx_encode(texts, which='vae_text'))
    vae = net.vae["text"]
    ids, lengths = vae.tokenize(texts)
    assert lengths == [10, 8, 2] and ids[0, :10].tolist() == [101] + [104 + words.index(w) for w in
                                                                    ("a", "red", "bus", "on", "a", "wet", "street", ".")] + [102]
    g = torch.Generator().manual_seed(41)
    c, u = torch.randn(3, 257, 768, generator=g) * 0.5, torch.zeros(3, 257, 768)
    with torch.no_grad():
        x, _ = DDIMSampler(net).sample(
            steps=10, shape=[3, 768], x_info={"type": "text", "x0": z, "x0_forward_timesteps": 4},
            c_info={"type": "image", "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                    "unconditional_guidance_scale": 7.5}, verbose=False, eta=0.)
    assert x.shape == (3, 768) and torch.isfinite(x).all()
    (vocab_dir / "gpt2-vocab.json").write_text(json.dumps({("Ġw%d" % i): i for i in range(50257)}), encoding="utf-8")
    torch.manual_seed(5)
    out = net.vae_decode(x, which='text', temperature=1)
    assert isinstance(out, list) and len(out) == 3 and all(isinstance(t, str) for t in out)
    print("[textenc] encode -> DDIM -> decode texts:", out)
