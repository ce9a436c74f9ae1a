"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/text_filter.npz from the UNMODIFIED reference's top_k_top_p_filtering
(lib/model_zoo/optimus.py:690-719), run on the CPU over seeded 50260-wide logit rows and the grid below.

    python oracle/make_text_filter_golden.py

Per (row, top_k, top_p, temperature) the fixture keeps what the reference kept: the count, the boundary value (the smallest kept
l), the sum of the indices of the kept tokens above the boundary (which tokens), how many tokens tied at the boundary it kept,
and its fp32 exclusive mass (the shifted cumsum) at the last kept and the first removed survivor, so a test can tell a real
mismatch from an fp32-versus-fp64 rounding case at the boundary.

The generator asserts that oracle/text_filter_oracle.filter_keep_mask keeps the same tokens above the boundary and the same
number of tied tokens at it, on every case, apart from tokens whose fp32 exclusive mass lies within NEAR of top_p.  Which of the
tied tokens are kept is not compared: over 50260 entries the reference's torch.sort(descending=True) is not stable, and the order
it gives equal values is neither ascending nor descending index (the 0.5-grid row shows it), so no rule reproduces it.  The
restatement, like the kernel, takes them in ascending index.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
V = 50260
TOP_K = (0, 1, 40, 50260, 60000)
TOP_P = (0.0, 0.5, 0.9, 0.999)
TEMPERATURE = (0.7, 1.0, 1.3)
NEAR = 1e-5
ROW_NAMES = ("seeded 0", "seeded 1", "seeded 2", "seeded 3", "ties at the k-th value and at the max",
             "logits on a 0.5 grid: ties at every nucleus boundary", "the top token alone exceeds top_p")


def filter_rows():
    """fp32 [7, V] logit rows, deterministic from a CPU generator (see ROW_NAMES)."""
    g = torch.Generator().manual_seed(4242)
    rows = [torch.randn(V, generator=g) * 3 for _ in range(4)]
    x = torch.randn(V, generator=g) * 3
    order = x.argsort(descending=True)
    x[order[36:44]] = x[order[39]].item()     # the 40th largest shared by ranks 36..43: top_k=40 keeps 44
    x[order[1]] = x[order[0]].item()          # a tie at the max: top_k=1 keeps 2
    rows.append(x)
    rows.append(torch.round(torch.randn(V, generator=g) * 6) / 2)
    x = torch.randn(V, generator=g)
    x[12345] = 40.0
    rows.append(x)
    return torch.stack(rows).float()


def reference_fp32_exclusive(ref_filter, l, top_k):
    """The reference's own nucleus quantities on row l after its top-k cut: the fp32 cumsum of the sorted softmax shifted right
    by one (the mass before each sorted position), and the sorted values."""
    f = ref_filter(l.clone(), top_k=top_k, top_p=0.0)
    s = torch.sort(f, descending=True).values
    cum = torch.cumsum(torch.softmax(s, -1), -1)
    return torch.cat([torch.zeros(1), cum[:-1]]), s


def main():
    sys.path.insert(0, ROOT)
    from oracle.text_dec_oracle import load_reference_optimus
    from oracle.text_filter_oracle import filter_keep_mask, scaled_logits
    _, optimus = load_reference_optimus()
    ref_filter = optimus.top_k_top_p_filtering
    rows = filter_rows()
    shape = (rows.shape[0], len(TOP_K), len(TOP_P), len(TEMPERATURE))
    out = {n: np.zeros(shape, dt) for n, dt in (("kept", np.int64), ("boundary", np.float32), ("above_index_sum", np.int64),
                                                  ("ties_kept", np.int64), ("excl_last", np.float32), ("excl_next", np.float32))}
    exempt = 0
    for r in range(rows.shape[0]):
        for t, temp in enumerate(TEMPERATURE):
            l = scaled_logits(rows[r], temp)
            for a, k in enumerate(TOP_K):
                for b, p in enumerate(TOP_P):
                    keep_ref = torch.isfinite(ref_filter(l.clone(), top_k=k, top_p=p))
                    keep = filter_keep_mask(l, k, p)
                    excl, s = reference_fp32_exclusive(ref_filter, l, k)
                    n = int(keep_ref.sum())
                    nucleus = 0.0 < p < 1.0
                    v = l[keep_ref].min()
                    out["kept"][r, a, b, t] = n
                    out["boundary"][r, a, b, t] = float(v)
                    out["above_index_sum"][r, a, b, t] = int((keep_ref & (l > v)).nonzero().sum())
                    out["ties_kept"][r, a, b, t] = int((keep_ref & (l == v)).sum())
                    out["excl_last"][r, a, b, t] = float(excl[n - 1]) if nucleus else 0.0
                    out["excl_next"][r, a, b, t] = float(excl[n]) if nucleus and n < V and torch.isfinite(s[n]) else np.inf
                    off = l != v
                    if int(keep.sum()) != n or not torch.equal(keep & off, keep_ref & off):
                        near = set(s[(excl - np.float32(p)).abs() < NEAR].tolist())
                        diff = l[(keep != keep_ref) & off].tolist() + ([float(v)] if int(keep.sum()) != n else [])
                        assert nucleus and all(x in near for x in diff), (ROW_NAMES[r], k, p, temp, int(keep.sum()), n)
                        exempt += 1
    print(f"restatement == reference on {rows.shape[0] * len(TOP_K) * len(TOP_P) * len(TEMPERATURE) - exempt} cases, "
          f"{exempt} exempt (boundary tokens within {NEAR} of top_p)")
    out.update(row_sum=rows.double().sum(-1).numpy(), top_k=np.array(TOP_K, np.int64), top_p=np.array(TOP_P, np.float64),
               temperature=np.array(TEMPERATURE, np.float64))
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "text_filter.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
