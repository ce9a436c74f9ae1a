"""Semantic/style disentanglement, CPU side: the oracle against the golden made with the reference's own decompose / adjust_rank,
the host factor schedule against the reference's in-place scaling of S, and the argument checks of vdb_rank_adjust_f32."""
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLD, "disentangle.npz")))


def test_oracle_fp32_reproduces_reference_golden(gold):
    """Same algorithm, same torch ops, same R: the fp32 oracle is the reference up to round-off.  The fp32 rounding of the 201
    QRs depends on the CPU's BLAS / LAPACK kernels (2.6e-5 apart between two x86 machines on the Gaussian input, as large as the
    fp32 result's own error), so the bound is twice that error, measured against the fp64 oracle, plus 1e-6 of the scale.
    The fixture holds each output as 256 sampled elements and the norms of all 256 token rows; a row norm moves by at most
    sqrt(768) times the largest element difference."""
    from lib.model_zoo.disentangle import adjust_rank
    from oracle.disentangle_oracle import digest, golden_inputs, rank_adjust
    R = torch.from_numpy(gold["R"].astype(np.float32))
    idx = torch.from_numpy(gold["sample_idx"].astype(np.int64))
    xs = golden_inputs()
    assert [digest(x) for x in xs] == list(gold["x_sha256"]), "the regenerated inputs are not the ones the golden was made from"
    for a, x in enumerate(xs):
        for b, lvl in enumerate(gold["lvls"]):
            f = adjust_rank().factors(float(lvl))
            out, S = rank_adjust(x, R, f.astype(np.float32), lvl < 0.5, dtype=torch.float32)
            out64, S64 = rank_adjust(x, R, f, lvl < 0.5, dtype=torch.float64)
            ref, ref_norm, ref_s = gold["out_sample"][a, b], gold["out_rownorm"][a, b], gold["s_before"][a, b]
            e32 = (out.double() - out64).abs().max().item()
            bound = 2 * e32 + 1e-6 * out64.abs().max().item()
            assert np.abs(out[0].flatten()[idx].numpy() - ref).max() <= bound, (a, lvl)
            norm = out[0].double().norm(dim=-1).numpy()
            assert np.abs(norm - ref_norm).max() <= np.sqrt(768) * bound + 1e-6 * ref_norm.max(), (a, lvl)
            e32_s = (S.double() - S64).abs()[0].numpy()
            assert (np.abs(S[0].numpy().astype(np.float64) - ref_s) <= 2 * e32_s + 1e-6 * ref_s).all(), (a, lvl)


def test_factor_schedule_matches_reference_scaling(gold):
    from lib.model_zoo.disentangle import adjust_rank
    for a in range(len(gold["x_sha256"])):
        for b, lvl in enumerate(gold["lvls"]):
            ratio = gold["s_after"][a, b].astype(np.float64) / gold["s_before"][a, b]
            f = adjust_rank().factors(float(lvl))
            np.testing.assert_allclose(f, ratio, rtol=1e-6, atol=1e-7, err_msg=f"lvl {lvl}")
            assert (f >= 0).all() and (f <= 1).all()
    assert np.array_equal(adjust_rank().factors(0.5), np.ones(20))


def test_rank_adjust_argument_checks_without_gpu():
    """Refused before any launch: VDB_ERR_INVALID for missing pointers / counts, VDB_ERR_UNSUPPORTED for other shapes (the fake
    addresses below are never dereferenced)."""
    import __graft_entry__ as g
    g.build()
    from vdb200._lib import lib
    x, R, f, out = 0x10000, 0x20000, 0x30000, 0x40000
    call = lambda x=x, n=1, m=256, d=768, R=R, q=20, niter=100, f=f, out=out: lib.vdb_rank_adjust_f32(
        x, n, m, d, R, q, niter, f, 1, out, None, None, None, None)
    for kw in (dict(x=None), dict(R=None), dict(f=None), dict(out=None)):
        assert call(**kw) == 1 and b"rank_adjust: null pointer" in lib.vdb_last_error()
    assert call(n=0) == 1 and b"n_items = 0" in lib.vdb_last_error()
    assert call(niter=-1) == 1 and b"niter" in lib.vdb_last_error()
    assert call(out=0x40008) == 1 and b"16-byte aligned" in lib.vdb_last_error()
    for kw in (dict(m=321), dict(m=39), dict(d=512), dict(q=16), dict(n=65536)):
        assert call(**kw) == 3 and b"rank_adjust: (m, n, q)" in lib.vdb_last_error(), kw


def test_product_refuses_cpu_tensors():
    from lib.model_zoo.disentangle import adjust_rank, decompose
    x = torch.zeros(1, 256, 768)
    with pytest.raises(RuntimeError, match="no CPU path"):
        adjust_rank()(x, 0.25)
    with pytest.raises(RuntimeError, match="no CPU path"):
        decompose(x)
    assert adjust_rank()(x, 0.5) is x      # lvl 0.5 is the identity, as in the reference
