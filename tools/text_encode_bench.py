"""Optimus BERT text encoding on one GPU at full size (12 layers, width 768), synthetic weights.  For n = 4 and 16 sentences of
77 pieces (Lp 80) and of about 12 pieces (Lp 16), reports from CUDA events after warm-up: ms per encode call (token ids to z_mu,
i.e. encode() without the host tokenizer), launches per call, the weight bytes a call must read and the rate that makes against
3.35 TB/s (H100 SXM data sheet).  Prints the card name and power limit, read in the same run.
    python tools/text_encode_bench.py"""
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))
import torch  # noqa: E402
from lib.model_zoo.optimus import optimus_vae_next  # noqa: E402
from vdb200 import ops  # noqa: E402

HBM = 3.35e12
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card)
torch.manual_seed(0)
vae = optimus_vae_next(decoder=dict(config=dict(n_layer=1)), encoder=dict(config={})).to(dev).eval()
with torch.no_grad():
    for name, p in vae.encoder.named_parameters():
        if not name.endswith("LayerNorm.weight"):               # weights and biases; LayerNorm scales stay 1
            p.normal_(0.0, 0.02)
vae.invalidate_packed()
enc = vae.packed()["enc"]
wbytes = sum(t.numel() * t.element_size() for L in enc["layers"] for v in L.values()
             for t in (v if isinstance(v, tuple) else (v,)) if torch.is_tensor(t))
wbytes += sum(t.numel() * t.element_size() for t in (enc["w_pool"], enc["b_pool"], enc["w_mu"]))


def ragged(n, pieces, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = [pieces + 2] * n if pieces == 77 else [int(v) + 2 for v in torch.randint(pieces - 3, pieces + 4, (n,), generator=g)]
    ids = torch.zeros(n, max(lengths), dtype=torch.long)
    for r, L in enumerate(lengths):
        ids[r, 0], ids[r, L - 1] = 101, 102
        ids[r, 1:L - 1] = torch.randint(999, 28996, (L - 2,), generator=g)
    return ids, lengths


results = []
with torch.no_grad():
    for n in (4, 16):
        for pieces in (77, 12):
            ids, lengths = ragged(n, pieces, seed=n * 100 + pieces)
            for _ in range(3):
                vae.encode_ids(ids, lengths)                   # warm-up: kernel configuration, allocator
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            vae.encode_ids(ids, lengths)
            launches = ops.launch_count() - n0
            reps = 50
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                vae.encode_ids(ids, lengths)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            results.append(dict(card=card, sentences=n, pieces_max=max(lengths) - 2, Lp=(max(lengths) + 7) // 8 * 8,
                                ms_per_encode=round(ms, 3), launches_per_call=launches, weight_bytes=wbytes,
                                achieved_TBps=round(wbytes / (ms * 1e-3) / 1e12, 3),
                                share_of_3_35_TBps=round(wbytes / (ms * 1e-3) / HBM, 3)))
            print(json.dumps(results[-1]))
