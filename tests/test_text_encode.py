"""Optimus text encoder, CPU side: the fp32 oracle against the reference's golden, the WordPiece tokenizer against the reference's
BertTokenizer, the key layout, the VDB_TEXT_FLOWS configuration and the argument checks of the varlen attention entry point."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def enc_golden():
    from oracle.make_text_enc_golden import synth_encoder_state
    keys = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLD, "keys_text_enc.json"))).items()}
    return keys, synth_encoder_state(keys), dict(np.load(os.path.join(GOLD, "text_enc.npz")))


def test_oracle_matches_reference_golden():
    from oracle.text_enc_oracle import bert_latent_mu
    _, sd, gold = enc_golden()
    mu, pooled = bert_latent_mu(sd, torch.from_numpy(gold["ids"]), return_pooled=True)
    assert mu.shape == (6, 768) and int(gold["n_layer"]) == 2
    for out, ref in ((mu, gold["z_mu"]), (pooled, gold["pooled"])):
        ref = torch.from_numpy(ref)
        assert (out - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()     # fp32 against fp32: round-off only


def test_module_key_layout_matches_reference():
    """`encoder.*` names and shapes of a 2-layer build equal the reference's (fixture); the decoder's keys are unchanged."""
    from lib.model_zoo.optimus import optimus_vae_next
    keys, _, _ = enc_golden()
    dec_keys = {k: tuple(v) for k, v in json.load(open(os.path.join(GOLD, "keys_text_dec.json"))).items()}
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=2)), encoder=dict(args=dict(config=dict(num_hidden_layers=2))))
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k: v for k, v in ours.items() if k.startswith("encoder.")} == keys
    assert {k: v for k, v in ours.items() if not k.startswith("encoder.")} == dec_keys
    with pytest.raises(TypeError, match="list of sentences"):
        m.encode("a sentence")
    with pytest.raises(ValueError, match="max_length"):
        m.encode(["a sentence"], max_length=511)


def test_text_flows_config_carries_the_encoder(monkeypatch):
    from lib.cfg_helper import model_cfg_bank
    monkeypatch.setenv("VDB_TEXT_FLOWS", "1")
    vl = dict((n, c) for n, c in model_cfg_bank()("vd_four_flow_v1-0").args.vae_cfg_list)
    a = vl["text"].args
    assert a.encoder.type == "optimus_bert_connector"
    assert a.encoder.args.config.num_hidden_layers == 12 and a.encoder.args.config.layer_norm_eps == 1e-12
    assert a.tokenizer_encoder.args.vocab_file == "lib/model_zoo/optimus_models/vocab/bert-base-cased-vocab.txt"


def test_tokenizer_on_a_synthetic_vocabulary(tmp_path):
    from lib.model_zoo.optimus import BertWordPieceTokenizer, VocabularyMissingError
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "hello", "world", "##s", "un", "##aff", "##able", ",", "!", "é", "中", "文"]
    path = tmp_path / "vocab.txt"
    path.write_text("\n".join(vocab) + "\n", encoding="utf-8")
    t = BertWordPieceTokenizer(str(path))
    ids = {p: i for i, p in enumerate(vocab)}
    assert t.tokenize("Hello, Worlds!") == ["hello", ",", "world", "##s", "!"]
    assert t.tokenize("unaffable\x00\u200b xyz 中文") == ["un", "##aff", "##able", "[UNK]", "中", "文"]   # NUL, U+200B dropped
    assert t.tokenize("É x" + "a" * 101) == ["é", "[UNK]"]                # lowercased, accent kept; no piece for 'xaaa...'
    assert t.encode("hello world", max_length=1) == [ids["[CLS]"], ids["hello"], ids["[SEP]"]]
    assert t.encode("") == t.encode("  \t") == [ids["[CLS]"], ids["[SEP]"]]
    with pytest.raises(VocabularyMissingError, match="bert-base-cased-vocab.txt"):
        BertWordPieceTokenizer(str(tmp_path / "missing" / "bert-base-cased-vocab.txt")).encode("hello")


FIXED_SENTENCES = [
    "A man riding a horse on the beach.",
    "Hello, world! It's 5 o'clock -- isn't it?",
    "Café crème brûlée à la carte, naïve façade; ÅNGSTRÖM.",
    "東京タワーと北京の天安门 are landmarks; 한국어 텍스트.",
    "emoji 😀🚀 and symbols ™ © ® € £ ¥ § ¶ • …",
    "control\x00chars\x07and\x1b[0mescape\ttabs\nnewlines\r\n and \ufffd replacement \u200b zero width",
    "[CLS] [SEP] [PAD] [MASK] [UNK] look like special tokens",
    "unbelievably " + "x" * 105 + " long",
    " ".join(["supercalifragilistic", "antidisestablishmentarianism", "pneumonoultramicroscopic"] * 12),
    "a b c d e f g h i j k l m n o p q r s t u v w x y z " * 4,
    "",
    "!!!???...,,,;;;:::",
    "Mixed CASE WoRdS with Ümlauts and ÇEDILLAS",
    "numbers 3.14159 and 1,000,000 and 2nd 3rd",
    "\u00a0non\u00a0breaking\u00a0spaces\u3000ideographic",
    "the quick brown fox jumps over the lazy dog " * 10,
]


def _vocab_file():
    from oracle import ref_shims
    return os.path.join(ref_shims.REF, "lib", "model_zoo", "optimus_models", "vocab", "bert-base-cased-vocab.txt")


def _seeded_sentences(pieces, n=300, seed=13):
    """Sentences assembled from vocabulary pieces: words, continuations glued on, punctuation, odd spacing."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        words = []
        for _ in range(int(torch.randint(1, 40, (1,), generator=g))):
            w = pieces[int(torch.randint(0, len(pieces), (1,), generator=g))]
            if w.startswith("##") and words:
                words[-1] += w[2:]
            else:
                words.append(w.lstrip("#") or w)
        sep = [" ", " ", " ", "  ", "\t", ""][int(torch.randint(0, 6, (1,), generator=g))]
        out.append(sep.join(words))
    return out


def test_tokenizer_matches_reference():
    """ids of optimus_vae_next.encode's tokenization (lowercase, basic + WordPiece, truncate, [CLS] / [SEP]) equal the reference's."""
    from oracle import ref_shims
    if not ref_shims.available():
        pytest.skip("reference tree not present")
    from test_text_decode import reference_lib
    from oracle.text_enc_oracle import reference_bert_tokenizer, reference_encode_ids
    from lib.model_zoo.optimus import BertWordPieceTokenizer
    with reference_lib():
        tok = reference_bert_tokenizer()
    ours = BertWordPieceTokenizer(_vocab_file())
    pieces = [ln.rstrip("\n") for ln in open(_vocab_file(), encoding="utf-8")]
    pieces = [p for p in pieces if not (p.startswith("[") and p.endswith("]"))]
    texts = FIXED_SENTENCES + _seeded_sentences(pieces)
    for max_length in (77, 200):
        want = reference_encode_ids(tok, texts, max_length=max_length)
        for t, w in zip(texts, want):
            assert ours.encode(t, max_length=max_length) == w, (t, max_length)
    assert any(len(w) == 79 for w in reference_encode_ids(tok, FIXED_SENTENCES)), "some fixed sentence must be truncated"
    # whitespace only: the reference emits one of its special tokens, chosen by the order of a Python set (the hash seed);
    # this tokenizer encodes it as the empty sentence
    cls, sep = ours.encode("")
    specials = {ours._load()[s] for s in ("[UNK]", "[SEP]", "[PAD]", "[CLS]", "[MASK]")}
    for t in ("   ", "\t\n", "\u3000"):
        w = reference_encode_ids(tok, [t])[0]
        assert len(w) == 3 and w[0] == cls and w[2] == sep and w[1] in specials, (t, w)
        assert ours.encode(t) == [cls, sep]


def test_varlen_attention_checks_arguments_before_launch():
    """null / misaligned kv_len, d_head other than 64 and causal masking are refused (the fake addresses are never touched)."""
    from vdb200._lib import lib
    q, k, vt, out, kvl = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000

    def call(kv_len=kvl, d_head=64, causal=0, H=12):
        return lib.vdb_attention_varlen_bf16(q, 1536, 0, k, 1536, 768, vt, 160, out, 768, 2, H, 80, 80, 80, 80, d_head,
                                             d_head ** -0.5, causal, kv_len, None)
    for kw, rc, msg in ((dict(kv_len=None), 1, b"kv_len"), (dict(kv_len=kvl + 2), 1, b"kv_len"), (dict(causal=1), 1, b"causal"),
                        (dict(d_head=80), 3, b"d_head 64"), (dict(d_head=40), 3, b"d_head 64"),
                        (dict(d_head=160), 3, b"d_head 64")):
        assert call(**kw) == rc and msg in lib.vdb_last_error(), (kw, lib.vdb_last_error())
    # the checks shared with vdb_attention_bf16 still apply
    assert lib.vdb_attention_varlen_bf16(None, 1536, 0, k, 1536, 768, vt, 160, out, 768, 2, 12, 80, 80, 80, 80, 64, 0.125, 0,
                                         kvl, None) == 1
    assert lib.vdb_attention_varlen_bf16(q, 1536, 0, k, 1536, 768, vt, 160, out, 768, 2, 12, 80, 80, 80, 84, 64, 0.125, 0,
                                         kvl, None) == 1


def test_pooler_tanh_is_accepted_and_gelu_still_refused():
    from vdb200._lib import lib
    from vdb200 import ops
    x, w, out = 0x10000, 0x20000, 0x30000
    assert ops.ACT_TANH == 6
    assert lib.vdb_textdec_gemv(x, 4, 768, 768, None, None, 0.0, w, 64, 768, None, 7, 0, out, 64, None) == 1
    assert b"VDB_ACT_TANH" in lib.vdb_last_error()
    assert lib.vdb_textdec_gemv(x, 4, 768, 768, None, None, 0.0, w, 64, 768, None, 2, 0, out, 64, None) == 1
