"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/text_enc.npz and keys_text_enc.json from the UNMODIFIED reference's Optimus BERT
encoder (a 2-layer build of configs/model/optimus.yaml 'optimus_bert_encoder' with synthetic weights) on seeded token rows of
ragged lengths, masked as optimus_vae_next.encode masks them (attention_mask = ids > 0).

    python oracle/make_text_enc_golden.py
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
CLS_ID, SEP_ID, VOCAB = 101, 102, 28996
LENGTHS = (2, 79, 13, 40, 5, 64)      # [CLS] [SEP] only (the empty sentence), a full 77-piece row, and lengths in between


def golden_inputs():
    """Token rows int64 [6, 79] ([CLS] pieces [SEP], zero padded) and their lengths."""
    g = torch.Generator().manual_seed(2025)
    L = max(LENGTHS)
    ids = torch.zeros(len(LENGTHS), L, dtype=torch.long)
    for r, n in enumerate(LENGTHS):
        ids[r, 0], ids[r, n - 1] = CLS_ID, SEP_ID
        ids[r, 1:n - 1] = torch.randint(999, VOCAB, (n - 2,), generator=g)
    return ids, list(LENGTHS)


def synth_encoder_state(keys_shapes):
    """Synthetic weights keyed by the product's 'encoder.'-prefixed names."""
    from oracle import weights
    return {k: weights.tensor_for(k, s, WEIGHT_SEED) for k, s in keys_shapes.items()}


def main():
    sys.path.insert(0, ROOT)
    from oracle import text_enc_oracle as T
    net = T.build_reference_encoder(n_layer=N_LAYER)
    keys = {"encoder." + k: list(v.shape) for k, v in net.state_dict().items()}
    sd = synth_encoder_state(keys)
    res = net.load_state_dict({k[len("encoder."):]: v for k, v in sd.items()})
    assert not res.missing_keys and not res.unexpected_keys, res
    ids, lengths = golden_inputs()
    with torch.no_grad():
        pooled = net(ids, attention_mask=(ids > 0).float())[1].float()          # the reference's own forward
        mu, _ = net.linear(pooled).chunk(2, -1)
    out = dict(ids=ids.numpy(), lengths=np.asarray(lengths, dtype=np.int64), pooled=pooled.numpy(), z_mu=mu.float().numpy(),
               n_layer=np.int64(N_LAYER), weight_seed=np.int64(WEIGHT_SEED))
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "text_enc.npz"), **out)
    with open(os.path.join(GOLD, "keys_text_enc.json"), "w") as fh:
        json.dump(keys, fh, indent=0, sort_keys=True)
    print("wrote", os.path.join(GOLD, "text_enc.npz"), os.path.getsize(os.path.join(GOLD, "text_enc.npz")), "bytes")


if __name__ == "__main__":
    main()
