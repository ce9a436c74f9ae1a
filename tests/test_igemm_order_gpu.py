"""Both tile walks of igemm_kernel on the GPU, against the fp64 references and per-element bounds of test_igemm_coverage_gpu.

run_igemm walks the tiles N-fast when the launch is single-pass, has several N tiles and its A operand outweighs W (see
test_tile_schedule_order.n_fast_rule), and M-fast otherwise.  Each row states the order it must get (asserted through
ops.igemm_last_plan()["n_fast"]) and, for the multi-tile rows, that some CTA runs two tiles on different N tiles under that order
on the reported grid: then the bias / LayerNorm tables cached in shared memory are reloaded and the next tile's LayerNorm row
partials are prefetched along the N-fast walk.  BN (and the 256-row tile where asked) is forced, so the plan does not depend on
the SM count."""
from collections import defaultdict

import pytest

import test_igemm_coverage_gpu as cov
from test_tile_schedule_order import walk


def _case(cid, kind, bn, mode, n_fast, walk=True, ksplit=1, bm256=False, **kw):
    return dict(id=cid, kind=kind, bn=bn, mode=mode, n_fast=n_fast, walk=walk, ksplit=ksplit, bm256=bm256, **kw)


CASES = [
    # A (M x 256 channels after the K tail) outweighs W (N x K): N-fast, on every epilogue family
    _case("nfast-m3-bn64", "gemm", 64, 3, 1, M=1200, N=1056, K=200, bias="vec", resid=True),
    _case("nfast-m0-bn128-silu", "gemm", 128, 0, 1, M=3000, N=1064, K=200, bias="vec", resid=True, act=cov.ACT_SILU),
    _case("nfast-m0-bn160-rowbias", "gemm", 160, 0, 1, M=257 * 12, N=1056, K=200, bias="batch", rpb=257, resid=True),
    _case("nfast-m4-geglu", "gemm", 256, 4, 1, M=4000, N=17 * 256, K=200, bias="vec", act=cov.ACT_GEGLU),
    _case("nfast-m5-bn128", "ln", 128, 5, 1, M=3000, N=1056, K=200, parts=5),         # row partials prefetched a tile ahead
    _case("nfast-m5-bn64-parts20", "ln", 64, 5, 1, M=3000, N=1056, K=200, parts=20),  # ... and not
    _case("nfast-m5-cols-bn128", "ln", 128, 5, 1, M=3000, N=1056, K=200, parts=5, on_cols=True),
    _case("nfast-m6-geglu", "ln", 256, 6, 1, M=4000, N=17 * 256, K=200, parts=5, geglu=True),
    _case("nfast-m7-bn160", "stats", 160, 7, 1, M=3000, N=1056, K=200, bias="vec", resid=True),
    _case("nfast-conv-32x40", "conv", 64, 3, 1, B=8, H=32, W=40, C=64, N=320, cmode=0, bias="batch", resid=True),
    _case("nfast-conv-s2", "conv", 64, 3, 1, B=8, H=64, W=80, C=64, N=320, cmode=1, bias="vec"),
    _case("nfast-bm256-m3", "gemm", 160, 3, 1, bm256=True, M=6000, N=1056, K=200, bias="vec", resid=True),
    _case("nfast-bm256-m7", "stats", 160, 7, 1, bm256=True, M=6000, N=1056, K=200, bias="vec", resid=True),
    # M-fast: W outweighs A, split-K, or a single N tile
    _case("mfast-m3-bn64-wide", "gemm", 64, 3, 0, M=1200, N=2080, K=200, bias="vec", resid=True),
    _case("mfast-m5-bn256", "ln", 256, 5, 0, M=1200, N=16 * 256 + 96, K=200, parts=5),
    _case("mfast-splitk", "gemm", 64, 0, 0, walk=False, ksplit=4, M=2000, N=128, K=1288, bias="vec", resid=True),
    _case("mfast-one-n-tile", "gemm", 64, 3, 0, walk=False, M=3000, N=64, K=200, bias="vec", resid=True),
]


def n_tile_changes(grid, tiles_m, tiles_n, ksplit, n_fast):
    seq = defaultdict(list)
    for cta, _m, n, _k, _ in walk(grid, tiles_m, tiles_n, ksplit, n_fast):
        seq[cta].append(n)
    return any(len(s) >= 2 and len(set(s)) >= 2 for s in seq.values())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_tile_order(case, monkeypatch):
    from vdb200 import ops
    if case["bm256"]:
        for name in ("gemm", "gemm_ln", "conv3x3"):
            orig = getattr(ops, name)
            monkeypatch.setattr(ops, name, lambda *a, _orig=orig, bn=0, **kw: _orig(*a, bn=bn | ops.BM256, **kw))
    out, ref, atol, plan = cov.RUN[case["kind"]](case)
    want = dict(bm=256 if case["bm256"] else 128, bn=case["bn"], mode=case["mode"], n_fast=case["n_fast"])
    assert {k: plan[k] for k in want} == want, (case["id"], plan)
    assert (plan["ksplit"] > 1) == (case["ksplit"] > 1), plan
    if case["walk"]:
        assert plan["tiles_m"] * plan["tiles_n"] > plan["grid"], plan
        assert n_tile_changes(plan["grid"], plan["tiles_m"], plan["tiles_n"], plan["ksplit"], plan["n_fast"]), plan
    cov.check(out, ref, atol, 2.0 ** -8, case["id"])
