"""TEST INFRASTRUCTURE ONLY. fp64 restatement of the text sampler's top-k / nucleus cuts (top_k_top_p_filtering, reference
lib/model_zoo/optimus.py:690-719, as sample_single_sequence_conditional applies it at :662-688) and of the inverse-CDF pick over
the tokens they keep (vdb_textdec_sample_filtered).
"""
import numpy as np
import torch


def scaled_logits(logits, temperature):
    """fp32 logits / temperature, one IEEE fp32 division per element, as the sampling kernel computes l."""
    x = torch.as_tensor(logits).float().numpy()
    return torch.from_numpy((x / np.float32(temperature)).astype(np.float32))


def filter_keep_mask(l, top_k, top_p):
    """One row of scaled logits l (fp32 [V]) -> bool keep mask [V].
    top_k > 0 keeps l >= the k-th largest l, k = min(top_k, V) (ties kept).  Then, when 0 < top_p < 1, the survivors are ordered
    by descending l, ties in ascending index (a stable sort), and a survivor is kept when the fp64 softmax mass of the survivors
    before it is <= top_p (rounded to fp32: the reference compares an fp32 cumsum with it); the first is always kept."""
    l64 = torch.as_tensor(l).double()
    V = l64.numel()
    keep = torch.ones(V, dtype=torch.bool)
    if top_k > 0:
        keep = l64 >= torch.topk(l64, min(top_k, V)).values[-1]
    if 0.0 < top_p < 1.0:
        order, excl = exclusive_mass(l64, keep)
        ks = excl <= float(np.float32(top_p))
        ks[0] = True
        ks &= keep[order]
        keep = torch.zeros(V, dtype=torch.bool)
        keep[order] = ks
    return keep


def exclusive_mass(l, keep):
    """(order, excl): the stable descending order of l and, along it, the fp64 softmax mass of the kept tokens before each one."""
    l64 = torch.as_tensor(l).double()
    p = torch.where(keep, torch.exp(l64 - l64[keep].max()), torch.zeros_like(l64))
    p = p / p.sum()
    order = torch.sort(l64, descending=True, stable=True).indices
    ps = p[order]
    return order, torch.cumsum(ps, 0) - ps


def filtered_pick(l, keep, u):
    """The inverse-CDF pick over the kept tokens in vocabulary order, in fp64: for each u (fp64 [n]) the first index whose
    cumulative kept mass / total exceeds u -> (int64 picks [n], fp64 distance of each u to the nearest step of that CDF)."""
    l64 = torch.as_tensor(l).double()
    p = torch.where(keep, torch.exp(l64 - l64[keep].max()), torch.zeros_like(l64))
    cdf = p.cumsum(0)
    cdf = cdf / cdf[-1]
    last = int(keep.nonzero().max())
    u = torch.as_tensor(u).double()
    pick = torch.searchsorted(cdf, u, right=True).clamp_max(last)
    near = (cdf[keep][None, :] - u[:, None]).abs().amin(-1)
    return pick, near
