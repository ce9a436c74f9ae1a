"""TEST INFRASTRUCTURE ONLY. fp32 CPU restatement of the Optimus GPT-2 text decoder, plus the import of the unmodified reference's
decoder for oracle/make_text_golden.py.

gpt2_latent_logits recomputes the whole prefix at every call, like the reference's sampling loop (optimus.py:662-688), so it does
not share the product's KV-cache bookkeeping: GPT2ForLatentConnector_XX.forward(input_ids, past=z) with latent_as_gpt_emb and
latent_as_gpt_memory on (optimus_gpt2.py:870-994, 1070-1082).
"""
import math

import torch

DECODER_PREFIX = "decoder."


def _ln(x, g, b, eps):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, eps)


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * torch.pow(x, 3))))


@torch.no_grad()
def gpt2_latent_logits(sd, z, ids, n_head=12, eps=1e-5):
    """sd: decoder state dict ('transformer.*' keys, an optional 'decoder.' prefix is stripped); z fp32 [n, latent];
    ids int64 [n, L] (starting with <BOS>) -> fp32 logits [n, L, vocab] of every position."""
    sd = {(k[len(DECODER_PREFIX):] if k.startswith(DECODER_PREFIX) else k): v.float() for k, v in sd.items()}
    z, ids = z.float(), ids.long()
    n, L = ids.shape
    nl = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.h."))
    wte, wpe = sd["transformer.wte.weight"], sd["transformer.wpe.weight"]
    D = wte.shape[1]
    dh = D // n_head
    mem = (z @ sd["transformer.linear.weight"].t()).view(n, nl, D)        # slice i: key and value of position 0 in layer i
    emb = z @ sd["transformer.linear_emb.weight"].t()
    h = wte[ids] + wpe[torch.arange(1, L + 1)][None] + emb[:, None]       # past_length = 1: <BOS> sits at wpe[1]
    visible = torch.ones(L, L + 1).tril(diagonal=1).bool()                # query j sees the latent and tokens 0..j
    for i in range(nl):
        p = f"transformer.h.{i}."
        x = _ln(h, sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], eps)
        qkv = x @ sd[p + "attn.c_attn.weight"] + sd[p + "attn.c_attn.bias"]
        q, k, v = qkv.split(D, dim=-1)
        k = torch.cat([mem[:, i:i + 1], k], 1)
        v = torch.cat([mem[:, i:i + 1], v], 1)
        q = q.view(n, L, n_head, dh).transpose(1, 2)
        k = k.view(n, L + 1, n_head, dh).transpose(1, 2)
        v = v.view(n, L + 1, n_head, dh).transpose(1, 2)
        w = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
        w = w.masked_fill(~visible, float("-inf")).softmax(-1)
        a = (w @ v).transpose(1, 2).reshape(n, L, D)
        h = h + (a @ sd[p + "attn.c_proj.weight"] + sd[p + "attn.c_proj.bias"])
        x = _ln(h, sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], eps)
        m = _gelu_tanh(x @ sd[p + "mlp.c_fc.weight"] + sd[p + "mlp.c_fc.bias"])
        h = h + (m @ sd[p + "mlp.c_proj.weight"] + sd[p + "mlp.c_proj.bias"])
    h = _ln(h, sd["transformer.ln_f.weight"], sd["transformer.ln_f.bias"], eps)
    return h @ wte.t()


def load_reference_optimus():
    """The reference's lib.model_zoo.optimus module (unmodified), imported on CPU."""
    from oracle import ref_shims
    ns = ref_shims.load()       # the Optimus modules need nothing beyond ref_shims' stubs (their boto3 imports are commented out)
    with ref_shims._cwd(ref_shims.REF):
        import lib.model_zoo.optimus as optimus
    return ns, optimus


def build_reference_decoder(n_layer=None):
    """The reference's GPT2ForLatentConnector_XX from configs/model/optimus.yaml ('optimus_gpt2_decoder'), n_layer overridable."""
    from oracle import ref_shims
    ns, optimus = load_reference_optimus()
    with ref_shims._cwd(ref_shims.REF):
        cfg = ns.model_cfg_bank()("optimus_gpt2_decoder")
        if n_layer is not None:
            cfg.args.config.n_layer = n_layer
            cfg.args.config.num_hidden_layers = n_layer
        net = ns.get_model()(cfg, verbose=False)
    net.eval()
    return net


def reference_tokenizer():
    """The reference's GPT2Tokenizer with the three added tokens, as optimus_vae.__init__ sets it up (optimus.py:22-34)."""
    from oracle import ref_shims
    ns, optimus = load_reference_optimus()
    with ref_shims._cwd(ref_shims.REF):
        tok = ns.get_model()(ns.model_cfg_bank()("optimus_gpt2_tokenizer"), verbose=False)
    tok.add_special_tokens({'pad_token': '<PAD>', 'bos_token': '<BOS>', 'eos_token': '<EOS>'})
    return tok
