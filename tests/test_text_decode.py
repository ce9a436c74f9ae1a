"""Optimus text decoder, CPU side: the fp32 oracle against the reference's golden logits, the detokenizer against the reference's
GPT2Tokenizer, the C ABI's argument checks and the VDB_TEXT_FLOWS configuration."""
import contextlib
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def golden_setup():
    from oracle.make_text_golden import golden_inputs, synth_decoder_state
    keys = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLD, "keys_text_dec.json"))).items()}
    gold = dict(np.load(os.path.join(GOLD, "text_dec.npz")))
    return keys, synth_decoder_state(keys), gold


def check_against_golden(logits, gold, rel):
    """logits [n, L, V] vs the fixture's summaries, every error relative to the largest |logit| of that position."""
    logits = torch.as_tensor(logits).float().cpu()
    top_val, top_idx = torch.from_numpy(gold["top_val"]), torch.from_numpy(gold["top_idx"]).long()
    cols, cols_val = torch.from_numpy(gold["cols"]), torch.from_numpy(gold["cols_val"])
    scale = torch.maximum(top_val.abs().amax(-1), cols_val.abs().amax(-1))
    err_top = (logits.gather(-1, top_idx) - top_val).abs().amax(-1)
    err_cols = (logits[..., cols] - cols_val).abs().amax(-1)
    err_lse = (torch.logsumexp(logits, -1) - torch.from_numpy(gold["lse"])).abs()
    worst = max((err_top / scale).max().item(), (err_cols / scale).max().item(), (err_lse / scale).max().item())
    assert worst <= rel, f"worst error {worst:.3g} of max|logit| (allowed {rel:.3g})"
    return worst


def test_oracle_teacher_forced_logits_match_reference_golden():
    from oracle.text_dec_oracle import gpt2_latent_logits
    keys, sd, gold = golden_setup()
    sd["decoder.lm_head.weight"] = sd["decoder.transformer.wte.weight"]
    logits = gpt2_latent_logits(sd, torch.from_numpy(gold["z"]), torch.from_numpy(gold["ids"]))
    assert logits.shape == (3, 12, 50260)
    check_against_golden(logits, gold, rel=2e-5)       # fp32 against fp32: summation-order round-off only


@contextlib.contextmanager
def reference_lib():
    """The reference is imported as the package `lib`, like this project's drop-in: put this project's modules back afterwards."""
    ours = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    path = list(sys.path)
    try:
        yield
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(ours)
        sys.path[:] = path


def _vocab_path():
    from oracle import ref_shims
    return os.path.join(ref_shims.REF, "lib", "model_zoo", "optimus_models", "vocab", "gpt2-vocab.json")


def test_detokenizer_matches_reference_tokenizer():
    """decode -> split()[1:-1] -> join (optimus.py:759-762) on 300 seeded rows with added tokens and split UTF-8 byte sequences."""
    from oracle import ref_shims
    if not ref_shims.available():
        pytest.skip("reference tree not present")
    from oracle.text_dec_oracle import reference_tokenizer
    from lib.model_zoo.optimus import GPT2Detokenizer
    with reference_lib():
        tok = reference_tokenizer()
    ours = GPT2Detokenizer(_vocab_path())
    enc = json.load(open(_vocab_path(), encoding="utf-8"))
    multibyte = [i for t, i in enc.items() if any(ord(c) >= 0x100 and ord(c) not in range(0x100, 0x121) for c in t)][:2000]
    lone = [enc[c] for c in ("Ã", "â", "Ģ", "Ġ", "Ċ") if c in enc]   # bytes that begin / split sequences
    g = torch.Generator().manual_seed(5)
    for n in range(300):
        L = int(torch.randint(2, 30, (1,), generator=g))
        ids = torch.randint(0, 50260, (L,), generator=g).tolist()
        for j in range(L):
            u = float(torch.rand(1, generator=g))
            if u < 0.08:
                ids[j] = 50257 + int(torch.randint(0, 3, (1,), generator=g))
            elif u < 0.2 and lone:
                ids[j] = lone[int(torch.randint(0, len(lone), (1,), generator=g))]
            elif u < 0.3 and multibyte:
                ids[j] = multibyte[int(torch.randint(0, len(multibyte), (1,), generator=g))]
        ids = [50258] + ids + [50259]
        want = ' '.join(tok.decode(ids, clean_up_tokenization_spaces=True).split()[1:-1])
        assert ours.sentence(ids) == want, (n, ids)


def test_detokenizer_on_a_synthetic_vocabulary(tmp_path):
    from lib.model_zoo.optimus import GPT2Detokenizer, VocabularyMissingError, BOS_ID, EOS_ID, PAD_ID
    vocab = {"ĠHello": 0, "Ġworld": 1, "Ġ.": 2, "Ġdon": 3, "'t": 4, "Ã": 5, "©": 6}
    path = tmp_path / "gpt2-vocab.json"
    path.write_text(json.dumps(vocab), encoding="utf-8")
    d = GPT2Detokenizer(str(path))
    assert d.sentence([BOS_ID, 4, 1, EOS_ID]) == "world"                   # <BOS> glues onto a first word without a leading space
    assert d.sentence([BOS_ID, 0, 1, 2, EOS_ID]) == "Hello world."
    assert d.sentence([BOS_ID, 0, 5, 6, EOS_ID]) == "Helloé"              # two byte-level tokens form one UTF-8 character
    assert d.sentence([BOS_ID, 0, 5, PAD_ID, EOS_ID]) == "Hello� <PAD>"   # a split sequence decodes with errors='replace'
    with pytest.raises(VocabularyMissingError, match="gpt2-vocab.json"):
        GPT2Detokenizer(str(tmp_path / "missing" / "gpt2-vocab.json")).sentence([BOS_ID, 0, EOS_ID])


def test_text_decoder_entry_points_check_arguments_before_launch():
    """null, oversize and misaligned arguments return VDB_ERR_INVALID with a message (the fake addresses are never touched)."""
    from vdb200._lib import lib
    x, w, out, bad = 0x10000, 0x20000, 0x30000, 0x20008
    gemv = lambda x=x, R=4, K=768, ldx=768, W=w, N=2304, ldw=768, out=out: lib.vdb_textdec_gemv(
        x, R, K, ldx, None, None, 0.0, W, N, ldw, None, 0, 0, out, N, None)
    for kw, msg in ((dict(x=None), b"null"), (dict(W=None), b"null"), (dict(R=17), b"R <= 16"), (dict(R=0), b"R <= 16"),
                    (dict(K=4096, ldx=4096, ldw=4096), b"K <= 3072"), (dict(K=100, ldx=100, ldw=100), b"K % 32"),
                    (dict(W=bad), b"16-byte aligned"), (dict(ldw=772), b"ldw % 8"), (dict(out=x), b"alias")):
        assert gemv(**kw) == 1 and msg in lib.vdb_last_error(), (kw, lib.vdb_last_error())
    assert lib.vdb_textdec_gemv(x, 4, 768, 768, x + 4096, None, 1e-5, w, 64, 768, None, 0, 0, out, 64, None) == 1
    assert lib.vdb_textdec_gemv(x, 4, 768, 768, None, None, 0.0, w, 64, 768, None, 2, 0, out, 64, None) == 1
    step = 0x40000
    assert lib.vdb_textdec_attention(None, 2304, x, 768, out, out, 4, 12, 32, step, 0.125, out, 768, None) == 1
    assert lib.vdb_textdec_attention(x, 2304, x, 768, out, out, 17, 12, 32, step, 0.125, out, 768, None) == 1
    assert lib.vdb_textdec_attention(x, 2304, x, 768, out + 2, out, 4, 12, 32, step, 0.125, out, 768, None) == 1
    assert b"aligned" in lib.vdb_last_error()
    assert lib.vdb_textdec_embed(None, 33, step, x, 50260, x, 1024, 1, x, 4, 768, out, None) == 1
    assert lib.vdb_textdec_embed(x, 33, step, x, 50260, x, 1024, 1, x, 32, 768, out, None) == 1
    sample = lambda R=4, temp=1.0, seed=x, uniforms=None: lib.vdb_textdec_sample(
        x, R, 50260, 50260, temp, seed, uniforms, 32, None, 0, out, 33, out, out, step, 50259, 30, None, None)
    assert sample(R=17) == 1 and b"R <= 16" in lib.vdb_last_error()
    assert sample(temp=0.0) == 1 and b"temperature" in lib.vdb_last_error()
    assert sample(seed=None) == 1 and b"seed" in lib.vdb_last_error()
    assert sample(seed=x + 4) == 1 and b"8-byte aligned" in lib.vdb_last_error()
    assert lib.vdb_textdec_sample(None, 4, 50260, 50260, 1.0, x, None, 0, None, 0, out, 33, out, out, step, 50259, 30, None,
                                  None) == 1


def test_text_flows_config_carries_the_text_vae(monkeypatch):
    from lib.cfg_helper import model_cfg_bank
    bank = model_cfg_bank()
    with pytest.raises(KeyError):
        bank("optimus_v1")
    monkeypatch.delenv("VDB_TEXT_FLOWS", raising=False)
    assert [n for n, _ in bank("vd_four_flow_v1-0").args.vae_cfg_list] == ["image"]
    monkeypatch.setenv("VDB_TEXT_FLOWS", "1")
    vl = dict((n, c) for n, c in bank("vd_four_flow_v1-0").args.vae_cfg_list)
    assert set(vl) == {"image", "text"} and vl["text"].type == "optimus_vae_next"
    assert vl["text"].args.tokenizer_decoder.args.vocab_file == "lib/model_zoo/optimus_models/vocab/gpt2-vocab.json"


def test_module_key_layout_matches_reference_on_cpu():
    """Parameter and buffer names / shapes of the 2-layer module equal the reference's (fixture), lm_head tied to wte."""
    from lib.model_zoo.optimus import optimus_vae_next
    keys = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLD, "keys_text_dec.json"))).items()}
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=2)))
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert ours == keys
    assert m.decoder.lm_head.weight is m.decoder.transformer.wte.weight
    with pytest.raises(NotImplementedError, match="BERT"):
        m.encode(["a sentence"])
