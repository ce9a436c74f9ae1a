"""TEST INFRASTRUCTURE ONLY. fp32 CPU restatement of the Optimus BERT encoder, plus the import of the unmodified reference's encoder
and tokenizer for oracle/make_text_enc_golden.py and the tokenizer parity test.

bert_latent_mu is BertForLatentConnector_XX.forward(ids, attention_mask=(ids > 0)) followed by linear(pooled).chunk(2)[0]
(optimus_bert.py:1393-1437, optimus.py:740-741): post-LN BERT layers (LayerNorm eps 1e-12, erf GELU), the padding mask as the
reference's additive -10000, the pooler's tanh on the [CLS] row.
"""
import math

import torch

ENCODER_PREFIX = "encoder."


def _ln(x, g, b, eps):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)


@torch.no_grad()
def bert_latent_mu(sd, ids, n_head=12, eps=1e-12, return_pooled=False):
    """sd: encoder state dict (an optional 'encoder.' prefix is stripped); ids int64 [n, L], 0 = padding -> z_mu fp32 [n, latent]
    (and the pooled [CLS] features [n, 768] when return_pooled)."""
    sd = {(k[len(ENCODER_PREFIX):] if k.startswith(ENCODER_PREFIX) else k): v.float() for k, v in sd.items()}
    ids = ids.long()
    n, L = ids.shape
    nl = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layer."))
    e = "embeddings."
    h = sd[e + "word_embeddings.weight"][ids] + sd[e + "position_embeddings.weight"][:L][None] + sd[e + "token_type_embeddings.weight"][0]
    h = _ln(h, sd[e + "LayerNorm.weight"], sd[e + "LayerNorm.bias"], eps)
    D = h.shape[-1]
    dh = D // n_head
    mask = (1.0 - (ids > 0).float())[:, None, None, :] * -10000.0
    for i in range(nl):
        p = f"encoder.layer.{i}."
        lin = lambda x, name: x @ sd[p + name + ".weight"].t() + sd[p + name + ".bias"]
        heads = lambda t: t.view(n, L, n_head, dh).transpose(1, 2)
        q, k, v = (heads(lin(h, "attention.self." + w)) for w in ("query", "key", "value"))
        w = (q @ k.transpose(-1, -2)) / math.sqrt(dh) + mask
        a = (w.softmax(-1) @ v).transpose(1, 2).reshape(n, L, D)
        h = _ln(lin(a, "attention.output.dense") + h, sd[p + "attention.output.LayerNorm.weight"],
                sd[p + "attention.output.LayerNorm.bias"], eps)
        m = torch.nn.functional.gelu(lin(h, "intermediate.dense"))
        h = _ln(lin(m, "output.dense") + h, sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], eps)
    pooled = torch.tanh(h[:, 0] @ sd["pooler.dense.weight"].t() + sd["pooler.dense.bias"])
    lw = sd["linear.weight"]
    mu = pooled @ lw[:lw.shape[0] // 2].t()
    return (mu, pooled) if return_pooled else mu


def build_reference_encoder(n_layer=None):
    """The reference's BertForLatentConnector_XX from configs/model/optimus.yaml ('optimus_bert_encoder'), n_layer overridable."""
    from oracle import ref_shims
    from oracle.text_dec_oracle import load_reference_optimus
    ns, optimus = load_reference_optimus()
    with ref_shims._cwd(ref_shims.REF):
        cfg = ns.model_cfg_bank()("optimus_bert_encoder")
        if n_layer is not None:
            cfg.args.config.num_hidden_layers = n_layer
        net = ns.get_model()(cfg, verbose=False)
    net.eval()
    return net


def reference_bert_tokenizer():
    """The reference's BertTokenizer as optimus_vae builds it ('optimus_bert_tokenizer': cased vocabulary, do_lower_case false)."""
    from oracle import ref_shims
    from oracle.text_dec_oracle import load_reference_optimus
    ns, optimus = load_reference_optimus()
    with ref_shims._cwd(ref_shims.REF):
        tok = ns.get_model()(ns.model_cfg_bank()("optimus_bert_tokenizer"), verbose=False)
    return tok


def reference_encode_ids(tok, texts, max_length=77):
    """The token rows of optimus_vae_next.encode (optimus.py:730-738), the reference's own calls, as lists of ids."""
    rows = []
    for sentence in texts:
        pieces = tok.tokenize(sentence.lower())[0:max_length]
        rows.append(tok.add_special_tokens_single_sentence([tok._convert_token_to_id(t) for t in pieces]))
    return rows
