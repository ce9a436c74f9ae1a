"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/text_dec.npz and keys_text_dec.json from the UNMODIFIED reference's Optimus GPT-2
decoder (a 2-layer build of configs/model/optimus.yaml 'optimus_gpt2_decoder' with synthetic weights), teacher-forced on seeded
latents and seeded token rows.

    python oracle/make_text_golden.py

The fixture keeps, per position: the top-16 logits and their ids, the logsumexp over the vocabulary and a fixed set of 256
vocabulary columns, so it stays well under 1 MB.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
N_LAYER = 2
WEIGHT_SEED = 7
ROWS, LENGTH, TOPK, NCOLS = 3, 12, 16, 256


def golden_inputs():
    """Seeded latents [3, 768], token rows [3, 12] starting with <BOS> (with <PAD> / <EOS> mixed in) and the 256 fixed columns."""
    g = torch.Generator().manual_seed(2024)
    z = torch.randn(ROWS, 768, generator=g)
    ids = torch.randint(0, 50260, (ROWS, LENGTH), generator=g)
    ids[:, 0] = 50258
    ids[1, 5], ids[2, 7] = 50257, 50259
    cols = torch.randperm(50260, generator=g)[:NCOLS].sort().values
    cols[:3] = torch.tensor([50257, 50258, 50259])
    return z, ids, cols.sort().values


def synth_decoder_state(keys_shapes):
    """Synthetic weights keyed by the product's 'decoder.'-prefixed names (lm_head.weight is tied to wte and not drawn)."""
    from oracle import weights
    return {k: weights.tensor_for(k, s, WEIGHT_SEED) for k, s in keys_shapes.items()
            if not k.endswith((".attn.bias", "lm_head.weight"))}


def summarise(logits, cols):
    top = logits.topk(TOPK, dim=-1)
    return dict(top_val=top.values.numpy(), top_idx=top.indices.numpy().astype(np.int32),
                lse=torch.logsumexp(logits, -1).numpy(), cols_val=logits[..., cols].numpy())


def main():
    sys.path.insert(0, ROOT)
    from oracle import text_dec_oracle as T
    net = T.build_reference_decoder(n_layer=N_LAYER)
    keys = {"decoder." + k: list(v.shape) for k, v in net.state_dict().items()}
    sd = synth_decoder_state(keys)
    res = net.load_state_dict({k[len("decoder."):]: v for k, v in sd.items()}, strict=False)
    assert set(res.missing_keys) <= {k for k in net.state_dict() if k.endswith((".attn.bias", "lm_head.weight"))}, res.missing_keys
    assert net.lm_head.weight.data_ptr() == net.transformer.wte.weight.data_ptr()
    z, ids, cols = golden_inputs()
    with torch.no_grad():
        logits = net(input_ids=ids, past=z)[0].float()             # the reference's own forward, full prefix
    out = dict(z=z.numpy(), ids=ids.numpy(), cols=cols.numpy().astype(np.int64), n_layer=np.int64(N_LAYER),
               weight_seed=np.int64(WEIGHT_SEED), **summarise(logits, cols))
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "text_dec.npz"), **out)
    with open(os.path.join(GOLD, "keys_text_dec.json"), "w") as fh:
        json.dump(keys, fh, indent=0, sort_keys=True)
    print("wrote", os.path.join(GOLD, "text_dec.npz"), os.path.getsize(os.path.join(GOLD, "text_dec.npz")), "bytes")


if __name__ == "__main__":
    main()
