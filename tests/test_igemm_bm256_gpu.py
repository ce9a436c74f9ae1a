"""The 256-row instantiations of the implicit-GEMM kernel (BM 256 x BN 160, epilogue modes 3 and 7) against the fp64 references
and per-element bounds of test_igemm_coverage_gpu, with the tile forced (bn = 160 | ops.BM256) so that the plan does not depend
on the SM count; and the shape rule: the long-K GEMM of the 32x32 level takes the 256-row tile, the 64x64 and 16x16 levels do not.

Rows marked walk make some CTA run two tiles on different N tiles (bias table reloaded, two staging boxes rotating across
tiles); they have an M tail (M % 256), a K tail and a partial last N tile.  The conv rows put the 256-pixel box on grids it
hangs over (24 x 40: a 64 x 4 box), with one bias row per image, a residual, and the interleaved store of the folded upsample."""
import pytest
import torch

import test_igemm_coverage_gpu as cov

M_WALK, K_WALK, N_WALK = 2500, 200, 16 * 160 + 96      # 10 M tiles (the last one 196 rows) x 17 N tiles (the last one 96 columns)


def _case(cid, kind, mode, walk=False, **kw):
    return dict(id=cid, kind=kind, bn=160, mode=mode, walk=walk, ksplit=1, **kw)


CASES = [
    _case("m3-gemm", "gemm", 3, walk=True, M=M_WALK, N=N_WALK, K=K_WALK, bias="vec", resid=True),
    _case("m3-gemm-nobias", "gemm", 3, M=300, N=160, K=64),
    _case("m7-stats", "stats", 7, walk=True, M=M_WALK, N=N_WALK, K=K_WALK, bias="vec", resid=True),
    _case("m7-stats-noresid", "stats", 7, M=700, N=320, K=328, bias="vec"),
    _case("conv-24x40-batchbias", "conv", 3, B=3, H=24, W=40, C=64, N=320, cmode=0, bias="batch", resid=True),
    _case("conv-32x32", "conv", 3, B=2, H=32, W=32, C=128, N=192, cmode=0, bias="batch", resid=True),
    _case("conv-s2-24x40", "conv", 3, B=3, H=24, W=40, C=128, N=128, cmode=1, bias="vec"),
    _case("conv-up-p2", "conv", 3, B=2, H=16, W=16, C=64, N=320, cmode=9, bias="batch"),
]


def geometry(case):
    """(M tiles, N tiles) of a forced 256 x 160 launch (host mirror of set_tile_shape)"""
    if case["kind"] == "conv":
        s = 2 if case["cmode"] in (1, 2) else 1
        Wo, Ho, Bo = case["W"] // s, case["H"] // s, case["B"]
        TW = min(cov._pow2_ceil(Wo), 256)
        TH = min(cov._pow2_ceil(Ho), 256 // TW)
        TB = 256 // (TW * TH)
        tm = -(-Wo // TW) * -(-Ho // TH) * -(-Bo // TB)
    else:
        tm = -(-case["M"] // 256)
    return tm, -(-case["N"] // 160)


@pytest.fixture
def force_bm256(monkeypatch):
    from vdb200 import ops
    for name in ("gemm", "gemm_ln", "conv3x3"):
        orig = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _orig=orig, bn=0, **kw: _orig(*a, bn=bn | ops.BM256, **kw))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_bm256_instantiation(case, force_bm256):
    out, ref, atol, plan = cov.RUN[case["kind"]](case)
    tm, tn = geometry(case)
    want = dict(bm=256, bn=160, stages=4, mode=case["mode"], ksplit=1, tiles_m=tm, tiles_n=tn)
    assert {k: plan[k] for k in want} == want, plan
    if case["walk"]:
        assert cov.multi_tile_n_change(plan["grid"], tm, tn, 1), plan
    cov.check(out, ref, atol, 2.0 ** -8, case["id"])


@pytest.mark.gpu
def test_bm256_is_refused_where_its_epilogue_does_not_exist():
    from vdb200 import ops
    from vdb200._lib import VdbError
    a, w = cov.rnd(512, 128, seed=1), cov.rnd(320, 128, seed=2)
    for kw in (dict(act=cov.ACT_SILU), dict(out_dtype=torch.float32), dict(bn=128 | ops.BM256)):
        with pytest.raises(VdbError):
            ops.gemm(a, w, **{"bn": 160 | ops.BM256, **kw})


@pytest.mark.gpu
def test_shape_rule_takes_256_rows_on_the_32x32_level_only():
    """ff2 of the 32x32 level at batch 8 (M 8192, N 640, K 2560, + residual): 128 tiles of 256 x 160 are one wave on the 132
    SMs of an H100 and the model prefers them.  At the 64x64 level (M 32768, N 320) they would be two waves, at the 16x16 level
    (M 2048, N 1280) 64 tiles would leave half the SMs idle: both stay on 128 rows.  All against fp64."""
    mid = dict(id="auto-32x32-ff2", kind="gemm", bn=0, mode=3, walk=False, ksplit=0, M=8192, N=640, K=2560, bias="vec", resid=True)
    out, ref, atol, plan = cov.run_gemm(mid)
    assert (plan["bm"], plan["bn"], plan["mode"], plan["tiles_m"], plan["tiles_n"]) == (256, 160, 3, 32, 4), plan
    cov.check(out, ref, atol, 2.0 ** -8, mid["id"])
    for cid, M, N, K, tm in (("auto-64x64-ff2", 32768, 320, 1280, 256), ("auto-16x16", 2048, 1280, 1280, 16)):
        out, ref, atol, plan = cov.run_gemm(dict(mid, id=cid, M=M, N=N, K=K))
        assert (plan["bm"], plan["bn"], plan["tiles_m"]) == (128, 160, tm), plan
        cov.check(out, ref, atol, 2.0 ** -8, cid)
