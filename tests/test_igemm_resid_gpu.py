"""The residual of the TMA-store epilogues (modes 3 and 7), which is TMA-loaded into the staging boxes its output leaves from.

Every row runs the launch twice on the same inputs: once into a fresh output, checked against the fp64 reference and bounds of
test_igemm_coverage_gpu, and once in place (out == resid), which must give the same bits: each box is loaded before the output
of the same chunk is stored over it.  The rows cover 2, 4, 5 and 8 chunks per tile against 4 boxes (BN 64 / 128 / 160 / 256),
the 256-row tile (2 boxes, 2 x 5 chunks per tile), M tails (rows past the output are zero-filled by the load and clipped by the
store), several tiles per CTA in both tile orders, the LayerNorm-statistics epilogue and a conv geometry whose box spans
several image rows and images."""
import pytest
import torch

import test_igemm_coverage_gpu as cov


def _case(cid, kind, bn, mode, bm256=False, **kw):
    return dict(id=cid, kind=kind, bn=bn, mode=mode, walk=False, ksplit=1, bm256=bm256, resid=True, **kw)


CASES = [
    _case("m3-bn64-nfast", "gemm", 64, 3, M=1200, N=1056, K=200, bias="vec"),
    _case("m3-bn128-mfast", "gemm", 128, 3, M=1200, N=4128, K=200, bias="vec"),
    _case("m3-bn160-nfast", "gemm", 160, 3, M=3000, N=1056, K=200, bias="vec"),
    _case("m3-bn256-mfast", "gemm", 256, 3, M=1200, N=4192, K=200, bias="vec"),
    _case("m3-bn160-nobias", "gemm", 160, 3, M=333, N=320, K=64),
    _case("m7-bn160", "stats", 160, 7, M=3000, N=1056, K=200, bias="vec"),
    _case("m7-bn64", "stats", 64, 7, M=1200, N=2080, K=200, bias="vec"),
    _case("bm256-m3", "gemm", 160, 3, bm256=True, M=6000, N=1056, K=200, bias="vec"),
    _case("bm256-m7", "stats", 160, 7, bm256=True, M=2500, N=2656, K=200, bias="vec"),
    _case("conv-24x40", "conv", 64, 3, B=3, H=24, W=40, C=64, N=320, cmode=0, bias="batch"),
    _case("conv-12x8", "conv", 160, 3, B=5, H=12, W=8, C=128, N=320, cmode=0, bias="vec"),
    _case("conv-bm256-32x32", "conv", 160, 3, bm256=True, B=2, H=32, W=32, C=128, N=192, cmode=0, bias="batch"),
]


def _run(case, inplace):
    """(out, ref, atol, plan, stats) of one launch; in place: out is the residual tensor itself"""
    from vdb200 import ops
    bn = case["bn"] | (ops.BM256 if case["bm256"] else 0)
    if case["kind"] == "conv":
        B, H, W, C, N = case["B"], case["H"], case["W"], case["C"], case["N"]
        x, w = cov.rnd(B, H, W, C, seed=1), cov.rnd(N, 9 * C, seed=2, scale=(9 * C) ** -0.5)
        b, bstride, _ = cov._bias(dict(case, rpb=H * W), B * H * W, N, 3)
        r = cov.rnd(B, H, W, N, seed=4)
        r0 = r.clone()
        out = ops.conv3x3(x, w, bias=b, bias_bstride=bstride, resid=r, out=r if inplace else None, mode=0, bn=bn, ksplit=1)
        plan = ops.igemm_last_plan()
        xc = cov._im2col64(x, 0)
        pre = cov.mm64(xc, w) + cov._bias_rows(b, bstride, H * W, B * H * W)
        atol = 4 * 9 * C * cov.U * cov.rss64(xc, w) + 2 * cov.U * pre.abs() + 2.0 ** -20 * r0.double().view(-1, N).abs()
        return out.view(-1, N), pre + r0.double().view(-1, N), atol, plan, None
    M, N, K = case["M"], case["N"], case["K"]
    a, w = cov.rnd(M, K, seed=1), cov.rnd(N, K, seed=2, scale=K ** -0.5)
    b, _, _ = cov._bias(case, M, N, 3)
    r = cov.rnd(M, N, seed=4)
    r0 = r.clone()
    stats = None
    if case["kind"] == "stats":
        stats = ops.ln_stats_buffer(M, N, a.device)
        out, _ = ops.gemm_ln(a, w, bias=b, resid=r, out=r if inplace else None, stats_out=stats, bn=bn)
    else:
        out = ops.gemm(a, w, bias=b, resid=r, out=r if inplace else None, bn=bn, ksplit=1)
    plan = ops.igemm_last_plan()
    pre = cov.mm64(a, w) + (b.double()[None, :] if b is not None else 0.0)
    atol = 4 * K * cov.U * cov.rss64(a, w) + 2 * cov.U * pre.abs() + 2.0 ** -20 * r0.double().abs()
    return out, pre + r0.double(), atol, plan, stats


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_residual_through_the_staging_boxes(case):
    out, ref, atol, plan, stats = _run(case, inplace=False)
    assert (plan["bm"], plan["bn"], plan["mode"], plan["ksplit"]) == (256 if case["bm256"] else 128, case["bn"], case["mode"], 1), plan
    cov.check(out, ref, atol, 2.0 ** -8, case["id"])
    out_ip, _, _, plan_ip, stats_ip = _run(case, inplace=True)
    assert plan_ip == plan
    assert torch.equal(out_ip, out), f"{case['id']}: in place (out == resid) differs from a separate output"
    if stats is not None:
        parts = 2 * plan["tiles_n"]
        assert torch.equal(stats_ip[:parts], stats[:parts]), f"{case['id']}: LayerNorm statistics differ in place"
