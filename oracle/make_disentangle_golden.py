"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/disentangle.npz from the UNMODIFIED reference's decompose + adjust_rank
(app.py:48-127).  Importing app.py would load a model and start Gradio, so the two definitions are taken from its syntax tree and
executed alone.  torch.randn is patched for the duration of each call so the Gaussian start is a fixed R; decompose is wrapped to
record S before the in-place scaling of adjust_rank and after it.

The inputs are oracle.disentangle_oracle.golden_inputs() (a Gaussian and a spectrally gapped [1, 256, 768] matrix, regenerated
from their seed); the fixture keeps their SHA-256 so a test notices if they ever come out different.  The start R is stored
(fp16-representable values).  To keep the fixture small, each output is stored as the norms of all 256 token rows plus 256
elements at fixed seeded positions; S before / after are stored in full.

    python oracle/make_disentangle_golden.py
"""
import ast
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.disentangle_oracle import digest, golden_inputs  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
APP = os.path.join("/root/reference", "app.py")
LVLS = (0.0, 0.1, 0.25, 0.4, 0.6, 0.75, 0.9, 1.0)
N_SAMPLE = 256
M, D, Q = 256, 768, 20


def reference_functions():
    """decompose and adjust_rank of app.py, executed from its syntax tree only."""
    tree = ast.parse(open(APP).read())
    defs = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in ("decompose", "adjust_rank")]
    assert len(defs) == 2
    ns = {"torch": torch, "np": np}
    exec(compile(ast.Module(body=defs, type_ignores=[]), APP, "exec"), ns)
    return ns


def run_reference(ns, x, R, lvl):
    rec = {}
    decompose = ns["decompose"]

    def wrapped(x, q=20, niter=100):
        u, s, v, x_mean, x_remain = decompose(x, q=q, niter=niter)
        rec["before"], rec["s"] = s.clone(), s
        return u, s, v, x_mean, x_remain

    ns["decompose"] = wrapped
    randn = torch.randn
    torch.randn = lambda *a, **k: R.clone()
    try:
        out = ns["adjust_rank"]()(x, lvl)
    finally:
        torch.randn = randn
        ns["decompose"] = decompose
    return out, rec["before"], rec["s"]


def main():
    ns = reference_functions()
    R = torch.randn(M, Q, generator=torch.Generator().manual_seed(5)).half().float()
    xs = golden_inputs()
    idx = torch.randperm(M * D, generator=torch.Generator().manual_seed(6))[:N_SAMPLE].sort().values
    sample = np.zeros((len(xs), len(LVLS), N_SAMPLE), np.float32)
    rownorm = np.zeros((len(xs), len(LVLS), M), np.float32)
    before = np.zeros((len(xs), len(LVLS), Q), np.float32)
    after = np.zeros_like(before)
    for a, x in enumerate(xs):
        for b, lvl in enumerate(LVLS):
            o, s0, s1 = run_reference(ns, x, R, lvl)
            sample[a, b], rownorm[a, b] = o[0].flatten()[idx].numpy(), o[0].double().norm(dim=-1).float().numpy()
            before[a, b], after[a, b] = s0[0].numpy(), s1[0].numpy()
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "disentangle.npz")
    np.savez_compressed(path, x_sha256=np.asarray([digest(x) for x in xs]), R=R.half().numpy(), lvls=np.asarray(LVLS),
                        sample_idx=idx.numpy().astype(np.int32), out_sample=sample, out_rownorm=rownorm, s_before=before,
                        s_after=after)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
