"""Every instantiation of the implicit-GEMM kernel (igemm.cu), and the state it carries from one tile to the next, against an
fp64 reference.

The launcher compiles 18 instantiations: BN in {64, 128, 160, 256} x epilogue modes {0, 3, 5, 7}, plus BN 256 x the GEGLU
modes {4, 6}.  Each row of CASES names the (BN, MODE) it means to reach and the inputs that get there; the test asserts the
plan the launcher reports (ops.igemm_last_plan) and compares every output element with the fp64 result on the same
bf16-rounded operands.  BN and ksplit are forced, so the plan does not depend on the SM count.

Rows marked walk=True must make some CTA run two or more tiles and change its N tile in between (checked on the reported
grid with test_tile_schedule.walk): that is when the bias / LayerNorm tables cached in shared memory are reloaded, the next
tile's row statistics are prefetched and the TMA-store staging alternates.  They also have an
M tail (M % 128 != 0), a K tail (K % 64 != 0) and, except for GEGLU (N % 256 == 0 by contract), a partial last N tile.
test_tile_schedule checks on the CPU that every instantiation has such a row at 132 SMs.

Tolerance, per element (U = 2^-24, fp32 unit roundoff; K = reduction length):
    |out - ref| <= rtol * |ref| + atol
  rtol = 2^-8 for bf16 outputs (round-to-nearest costs 2^-9, the rest is margin) and 2^-16 for fp32 outputs.
  atol for a plain GEMM element: 4 K U ||a_m * w_n||_2 (fp32 accumulation of K products whose running sums stay within a few
  times the root-sum-square of the products) times alpha and 1.25 for the activation's slope, plus 2^-20 (|pre| + |resid|)
  for the epilogue's fp32 roundings and fast-math activations.  The per-test docstrings add what their epilogue computes on
  top of that.  The cosine >= 0.999 check of test_kernels_gpu is kept as well.
"""
import math
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from test_tile_schedule import walk

DEV = "cuda"
U = 2.0 ** -24
STAGES = {64: 8, 128: 6, 160: 5, 256: 4}
ACT_NONE, ACT_SILU, ACT_GELU, ACT_QGELU, ACT_GEGLU = 0, 1, 2, 3, 4

# ---------------------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------------------
# The multi-tile rows: M 1200 (10 M tiles, the last one 48 rows), K 200 (four k-blocks, the last one 8 channels) and 17 N tiles,
# the last one partial: 170 tiles, so on 132 SMs CTAs 0..37 run a second tile on another N tile (and another M tile).
M_WALK, K_WALK = 1200, 200
N_WALK = {64: 16 * 64 + 32, 128: 16 * 128 + 32, 160: 16 * 160 + 96, 256: 16 * 256 + 96}     # N % 32 == 0
N_WALK_ODD = {64: 16 * 64 + 40, 128: 16 * 128 + 40, 160: 16 * 160 + 104, 256: 16 * 256 + 104}  # N % 32 == 8: mode 0 only
N_GEGLU = 17 * 256


def _case(cid, kind, bn, mode, walk=False, ksplit=1, **kw):
    return dict(id=cid, kind=kind, bn=bn, mode=mode, walk=walk, ksplit=ksplit, **kw)


CASES = []
for _bn, _act, _alpha in ((64, ACT_SILU, 1.0), (128, ACT_GELU, 1.0), (160, ACT_QGELU, 1.0), (256, ACT_NONE, 0.5)):
    # mode 0: activation / alpha / N % 32 != 0 keep the launch on the generic epilogue
    CASES.append(_case(f"m0-bn{_bn}", "gemm", _bn, 0, walk=True, M=M_WALK, N=N_WALK_ODD[_bn], K=K_WALK, bias="vec", resid=True,
                       act=_act, alpha=_alpha))
for _bn in (64, 128, 160, 256):
    CASES.append(_case(f"m3-bn{_bn}", "gemm", _bn, 3, walk=True, M=M_WALK, N=N_WALK[_bn], K=K_WALK, bias="vec", resid=True))
    CASES.append(_case(f"m5-bn{_bn}", "ln", _bn, 5, walk=True, M=M_WALK, N=N_WALK[_bn], K=K_WALK,
                       parts={64: 5, 128: 25, 160: 8, 256: 20}[_bn]))          # ln_parts <= 16: prefetched a tile ahead; > 16: not
    CASES.append(_case(f"m7-bn{_bn}", "stats", _bn, 7, walk=True, M=M_WALK, N=N_WALK[_bn], K=K_WALK, bias="vec", resid=_bn != 128))
CASES += [
    _case("m4-bn256", "gemm", 256, 4, walk=True, M=M_WALK, N=N_GEGLU, K=K_WALK, bias="vec", act=ACT_GEGLU),
    _case("m6-bn256", "ln", 256, 6, walk=True, M=M_WALK, N=N_GEGLU, K=K_WALK, parts=5, geglu=True),
    _case("m6-bn256-parts20", "ln", 256, 6, walk=True, M=M_WALK, N=N_GEGLU, K=K_WALK, parts=20, geglu=True),
    # mode 0 paths the rows above do not take
    _case("m0-f32-ntail", "gemm", 128, 0, M=1000, N=200, K=328, bias="vec", f32=True),
    _case("m0-bf16-n24", "gemm", 64, 0, M=300, N=24, K=72, bias="vec", resid=True, act=ACT_SILU),   # one chunk narrower than a box
    _case("m0-f32-silu-alpha", "gemm", 64, 0, walk=True, M=M_WALK, N=N_WALK_ODD[64], K=K_WALK, bias="vec", act=ACT_SILU, alpha=1.5, f32=True),
    # per-row bias whose 128-row tiles straddle two (or, at 77 rows, three) batch items: each row reads its own bias row; at 257 rows some
    # tiles lie inside one item and take the shared-memory bias row, reloaded per item
    _case("m0-rowbias77", "gemm", 64, 0, walk=True, M=77 * 13, N=N_WALK[64], K=K_WALK, bias="batch", rpb=77, resid=True),
    _case("m0-rowbias257", "gemm", 160, 0, walk=True, M=257 * 5, N=N_WALK[160], K=K_WALK, bias="batch", rpb=257, resid=True),
    # GEGLU with a per-row bias: tiles that straddle two of the 200-row items keep GEGLU on the generic epilogue
    _case("m0-geglu-rowbias200", "gemm", 256, 0, walk=True, M=200 * 6, N=N_GEGLU, K=K_WALK, bias="batch", rpb=200, act=ACT_GEGLU),
    # split-K: fp32 partials, then splitk_reduce_kernel adds the per-batch bias, activation and residual
    _case("m0-splitk-rowbias", "gemm", 128, 0, ksplit=4, M=320, N=640, K=1288, bias="batch", rpb=80, resid=True, act=ACT_SILU),
    _case("m0-splitk-f32", "gemm", 64, 0, ksplit=3, M=300, N=200, K=520, bias="vec", f32=True, act=ACT_GELU),
    # folded LayerNorm with the statistics on the output columns (the transposed V^T projection)
    _case("m5-cols-bn128", "ln", 128, 5, walk=True, M=M_WALK, N=N_WALK[128], K=K_WALK, parts=5, on_cols=True),
    _case("m5-cols-bn64-parts20", "ln", 64, 5, walk=True, M=M_WALK, N=N_WALK[64], K=K_WALK, parts=20, on_cols=True),
    # 3x3 convs.  The 8x8 UNet level's ResBlock conv1 (B 8, 1280 -> 1280, the time embedding as a per-batch bias): the tile box
    # is 8 x 8 x 2 images, so every tile straddles two bias rows (mode 0, per-row bias); with split-K the reduction adds that bias
    _case("conv-8x8-rb-ks1", "conv", 64, 0, ksplit=1, B=8, H=8, W=8, C=1280, N=1280, cmode=0, bias="batch"),
    _case("conv-8x8-rb-ks4", "conv", 160, 0, ksplit=4, B=8, H=8, W=8, C=1280, N=1280, cmode=0, bias="batch"),
    _case("conv-8x8-rb-auto", "conv", 0, 0, ksplit=0, B=8, H=8, W=8, C=1280, N=1280, cmode=0, bias="batch"),
    # non-power-of-two grids: the (TW, TH, TB) box hangs past the image; those rows are masked on store
    _case("conv-24x40-silu", "conv", 64, 0, walk=True, B=3, H=24, W=40, C=64, N=320, cmode=0, bias="vec", resid=True, act=ACT_SILU),
    _case("conv-24x40-batchbias", "conv", 64, 3, walk=True, B=3, H=24, W=40, C=64, N=320, cmode=0, bias="batch", resid=True),
    _case("conv-12x8", "conv", 128, 3, B=3, H=12, W=8, C=128, N=160, cmode=0, bias="batch", resid=True),
    _case("conv-s2-24x40", "conv", 64, 3, B=3, H=24, W=40, C=128, N=128, cmode=1, bias="vec"),
    _case("conv-s2vae-24x40-f32", "conv", 128, 0, B=1, H=24, W=40, C=64, N=96, cmode=2, bias="vec", f32=True),
    _case("conv-s2vae-12x8-b5", "conv", 64, 0, B=5, H=12, W=8, C=64, N=96, cmode=2, bias="batch"),
    # folded nearest-2x upsample + 3x3 conv (2x2 taps on the source image, one launch per output parity): modes 7..10 store the
    # parity straight into the interleaved [B, 2H, 2W, N] result through the output tensor map, modes 3..6 into a dense
    # [B, H, W, N] tensor; both run the TMA-store epilogue (plan mode 3)
    _case("conv-up-p0", "conv", 64, 3, B=3, H=12, W=20, C=64, N=96, cmode=7, bias="vec"),
    _case("conv-up-p1", "conv", 128, 3, B=3, H=12, W=20, C=128, N=160, cmode=8, bias="vec"),
    _case("conv-up-p2", "conv", 160, 3, B=2, H=16, W=16, C=64, N=320, cmode=9, bias="batch"),
    _case("conv-up-p3", "conv", 256, 3, B=3, H=12, W=20, C=64, N=320, cmode=10, bias="vec"),
    _case("conv-upc-p1", "conv", 64, 3, B=3, H=12, W=20, C=64, N=160, cmode=4, bias="batch", resid=True),
    _case("conv-upc-p2", "conv", 160, 3, B=2, H=24, W=40, C=128, N=320, cmode=5, bias="vec", resid=True),
]


# ---------------------------------------------------------------------------------------------------------------------------
# tile geometry (host mirror of vdb_gemm_bf16 / set_tile_shape, as far as a forced BN needs) and the tile-walk property
# ---------------------------------------------------------------------------------------------------------------------------
def _pow2_ceil(v):
    t = 1
    while t < v:
        t <<= 1
    return t


def tile_geometry(case):
    """-> (tiles_m, tiles_n, ksplit, k-blocks) of the launch a case makes with its forced BN / ksplit"""
    if case["kind"] == "conv":
        s = 2 if case["cmode"] in (1, 2) else 1
        Wo, Ho, Bo = case["W"] // s, case["H"] // s, case["B"]
        TW = min(_pow2_ceil(Wo), 128)
        TH = min(_pow2_ceil(Ho), 128 // TW)
        TB = 128 // (TW * TH)
        tiles_m = -(-Wo // TW) * -(-Ho // TH) * -(-Bo // TB)
        kb = (4 if case["cmode"] >= 3 else 9) * case["C"] // 64
    else:
        tiles_m = -(-case["M"] // 128)
        kb = -(-case["K"] // 64)
    tiles_n = -(-case["N"] // case["bn"])
    ks = max(case["ksplit"], 1)
    per = -(-kb // ks)
    return tiles_m, tiles_n, -(-kb // per), kb


def multi_tile_n_change(grid, tiles_m, tiles_n, ksplit):
    """some CTA runs >= 2 tiles and not all of them on one N tile"""
    seq = defaultdict(list)
    for cta, _m, n, _k in walk(grid, tiles_m, tiles_n, ksplit):
        seq[cta].append(n)
    return any(len(s) >= 2 and len(set(s)) >= 2 for s in seq.values())


# ---------------------------------------------------------------------------------------------------------------------------
# GPU side
# ---------------------------------------------------------------------------------------------------------------------------
def _ops():
    from vdb200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def rnd(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    return (torch.randn(*shape, generator=_gen(seed)) * scale).to(dtype).to(DEV)


def mm64(a, w):
    return a.double() @ w.double().t()


def rss64(a, w):
    """||a_m * w_n||_2 for every (m, n): the scale of the fp32 accumulation error"""
    return (a.double().square() @ w.double().square().t()).sqrt()


def act64(x, act):
    if act == ACT_SILU:
        return F.silu(x)
    if act == ACT_GELU:
        return F.gelu(x)
    if act == ACT_QGELU:
        return x * torch.sigmoid(1.702 * x)
    return x


def geglu64(h):
    """packed [M, 256 t + (value 0..127 | gate 128..255)] -> value * gelu(gate), [M, 128 t + j]; also returns (value, gate)"""
    M, N = h.shape
    hv = h.view(M, N // 256, 2, 128)
    val, gate = hv[:, :, 0, :].reshape(M, -1), hv[:, :, 1, :].reshape(M, -1)
    return val * F.gelu(gate), val, gate


def geglu_err(val, gate, e_val, e_gate):
    """error bound of value * gelu_fast(gate) given bounds on value and gate: first-order propagation (|gelu'| <= 1.13) plus
    the tanh-form GELU's distance from the erf form and tanh.approx's error, < 1e-3 |gate| in gelu(gate)"""
    return F.gelu(gate).abs() * e_val + val.abs() * (1.13 * e_gate + 1e-3 * gate.abs())


def check(out, ref, atol, rtol, what):
    out = out.double()
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs()
    lim = rtol * ref.abs() + atol
    bad = err > lim
    if bad.any():
        i = int((err - lim).argmax())
        idx = list(torch.unravel_index(torch.tensor(i), err.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of tolerance; worst at {[int(j) for j in idx]}: "
                             f"out {out.flatten()[i].item():.6g} ref {ref.flatten()[i].item():.6g} limit {lim.flatten()[i].item():.3g}")
    cos = F.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    assert cos >= 0.999, f"{what}: cosine {cos:.6f}"


def check_plan(case, plan):
    want = {"mode": case["mode"]}
    if case["bn"]:
        want["bn"] = case["bn"]
        want["stages"] = STAGES[case["bn"]]
    if case["ksplit"]:
        want["ksplit"] = tile_geometry(case)[2]
    got = {k: plan[k] for k in want}
    assert got == want, f"{case['id']}: launched {plan}, case expects {want}"
    if case["bn"]:
        tm, tn, _, _ = tile_geometry(case)
        assert (plan["tiles_m"], plan["tiles_n"]) == (tm, tn), (plan, tm, tn)
    if case["walk"]:
        assert multi_tile_n_change(plan["grid"], plan["tiles_m"], plan["tiles_n"], plan["ksplit"]), \
            f"{case['id']}: no CTA runs two tiles on different N tiles ({plan})"


def _bias(case, rows, N, seed):
    """fp32 bias [N] (vec) or one row per batch item [rows / rpb, N] (batch), with distinct rows so that a wrong row shows"""
    if case.get("bias") == "vec":
        return rnd(N, seed=seed, dtype=torch.float32), 0, 1
    if case.get("bias") == "batch":
        nb = -(-rows // case["rpb"])
        b = rnd(nb, N, seed=seed, dtype=torch.float32) + torch.arange(nb, device=DEV, dtype=torch.float32)[:, None]
        return b, N, case["rpb"]
    return None, 0, 1


def _bias_rows(b, bstride, rpb, rows):
    if b is None:
        return 0.0
    if bstride == 0:
        return b.double()[None, :]
    return b.double().repeat_interleave(rpb, 0)[:rows]


def run_gemm(case):
    """vdb_gemm_bf16: out = act(alpha (a w^T + bias)) + resid (GEGLU: value * gelu(gate) of the packed halves)."""
    ops = _ops()
    M, N, K, act, alpha = case["M"], case["N"], case["K"], case.get("act", 0), case.get("alpha", 1.0)
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    b, bstride, rpb = _bias(case, M, N, 3)
    n_out = N // 2 if act == ACT_GEGLU else N
    r = rnd(M, n_out, seed=4) if case.get("resid") else None
    f32 = case.get("f32", False)
    out = ops.gemm(a, w, bias=b, resid=r, act=act, alpha=alpha, bias_bstride=bstride, rows_per_batch=rpb, bn=case["bn"],
                   ksplit=case["ksplit"], out_dtype=torch.float32 if f32 else torch.bfloat16)
    plan = ops.igemm_last_plan()
    pre = mm64(a, w) + _bias_rows(b, bstride, rpb, M)
    e_pre = 4 * K * U * rss64(a, w) + 2 * U * pre.abs()
    if act == ACT_GEGLU:
        ref, val, gate = geglu64(pre)
        ev, eg = geglu64(e_pre)[1:]
        atol = geglu_err(val, gate, ev, eg)
    else:
        ref = act64(alpha * pre, act)
        atol = 1.25 * alpha * e_pre + 2.0 ** -20 * (alpha * pre).abs()
    if r is not None:
        ref = ref + r.double()
        atol = atol + 2.0 ** -20 * r.double().abs()
    return out, ref, atol, plan


def _ln_rows_input(rows, K, seed):
    """rows with their own mean in [-4, 4] and std in [0.5, 2]: |mean| / std up to 8, so the rank-1 correction cancels a lot"""
    g = _gen(seed)
    mu = torch.rand(rows, 1, generator=g) * 8 - 4
    sd = torch.rand(rows, 1, generator=g) * 1.5 + 0.5
    return (torch.randn(rows, K, generator=g) * sd + mu).to(torch.bfloat16).to(DEV)


def _stats_table(x, parts):
    """[parts, rows, 2] fp32 (sum, sum of squares) over `parts` near-equal column ranges of x, exact in fp64 then rounded"""
    xd = x.double()
    cols = torch.tensor_split(torch.arange(x.shape[1], device=DEV), parts)
    st = torch.stack([torch.stack([xd[:, c].sum(1), xd[:, c].square().sum(1)], -1) for c in cols])
    return st.float().contiguous()


def run_ln(case):
    """vdb_gemm_ln_bf16 consumer: out = rstd (x W'^T - mean s) + c from the raw x and per-range partial sums (ln_parts of them).
    Reference: LN(x) W'^T + c in fp64 (s = sum_k W'[n, k] exactly, then rounded to fp32 for the kernel).
    Bound, added to the plain-GEMM one (4 K U rstd ||x * w||_2) and doubled: the kernel sums the partials in fp32 and forms
    var = E[x^2] - mean^2, so rstd carries a relative error of (P + 4) U (1 + mean^2 / var) (the cancellation grows with
    |mean| / std) and mean one of (P + 4) U sqrt(mean^2 + var); both reach the output through |ref - c| and rstd |mean s|.
    GEGLU: the value / gate bounds propagate as in run_gemm."""
    ops = _ops()
    M, N, K, P, on_cols, geglu = case["M"], case["N"], case["K"], case["parts"], case.get("on_cols", False), case.get("geglu", False)
    if on_cols:          # out [M, N] = W0' LN(x)^T: A = prepared weights [M, K], B = x [N, K], statistics per output column
        w, x = rnd(M, K, seed=2, scale=K ** -0.5), _ln_rows_input(N, K, 1)
        a, bmat = w, x
    else:
        x, w = _ln_rows_input(M, K, 1), rnd(N, K, seed=2, scale=K ** -0.5)
        a, bmat = x, w
    s64 = w.double().sum(1)
    c = rnd(M if on_cols else N, seed=3, dtype=torch.float32)
    st = _stats_table(x, P)
    ln = ops.LnFold(st, P, K, 1e-5)
    if on_cols:
        out = ops.gemm_ln(a, bmat, ln=ln, colsum=s64.float(), on_cols=True, rowbias=c, bn=case["bn"])
    else:
        out = ops.gemm_ln(a, bmat, bias=c, act=ACT_GEGLU if geglu else ACT_NONE, ln=ln, colsum=s64.float(), bn=case["bn"])
    plan = ops.igemm_last_plan()
    xd = x.double()
    mean = xd.mean(1)
    var = xd.square().mean(1) - mean.square()
    rstd = (var + 1e-5).rsqrt()
    acc, rss = mm64(a, bmat), rss64(a, bmat)
    if on_cols:
        mean, var, rstd = mean[None, :], var[None, :], rstd[None, :]
        s, cc = s64[:, None], c.double()[:, None]
    else:
        mean, var, rstd = mean[:, None], var[:, None], rstd[:, None]
        s, cc = s64[None, :], c.double()[None, :]
    pre = rstd * (acc - mean * s) + cc
    e_pre = 2 * (rstd * 4 * K * U * rss + rstd * 4 * U * (mean * s).abs()
                 + (P + 4) * U * rstd * s.abs() * (mean.square() + var).sqrt()
                 + (P + 4) * U * (1 + mean.square() / var) * (pre - cc).abs()) + 2 * U * pre.abs()
    if geglu:
        ref, val, gate = geglu64(pre)
        ev, eg = geglu64(e_pre)[1:]
        return out, ref, geglu_err(val, gate, ev, eg), plan
    return out, pre, e_pre, plan


def run_stats(case):
    """vdb_gemm_ln_bf16 producer: out = a w^T + bias + resid, and per output row one (sum, sum of squares) partial per N tile and
    epilogue warp of the fp32 values before rounding.  Partial 2 n + s of a row holds the 32-column chunks c of N tile n with
    c % 2 == s (the two warps of a row quarter own alternate chunks; at BN 160 they swap which one takes the odd chunk every
    tile, but the partial slot follows the chunk).  Bound on a partial: the element bounds summed over its columns (times
    2 |ref| + bound for the squares) plus 40 U times the sum of |values| (fp32 sums over 32 columns, then over <= 4 chunks)."""
    ops = _ops()
    M, N, K, BN = case["M"], case["N"], case["K"], case["bn"]
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    b = rnd(N, seed=3, dtype=torch.float32)
    r = rnd(M, N, seed=4) if case.get("resid") else None
    stats = ops.ln_stats_buffer(M, N, a.device)
    stats.fill_(float("nan"))
    out, parts = ops.gemm_ln(a, w, bias=b, resid=r, stats_out=stats, bn=BN)
    plan = ops.igemm_last_plan()
    ref = mm64(a, w) + b.double()[None, :]
    e = 4 * K * U * rss64(a, w) + 2 * U * ref.abs()
    if r is not None:
        ref = ref + r.double()
        e = e + 2 * U * r.double().abs()
    tiles_n = -(-N // BN)
    assert parts == 2 * tiles_n, (parts, tiles_n)
    j = torch.arange(N, device=DEV)
    slot = (j // BN) * 2 + ((j % BN) // 32) % 2
    S = F.one_hot(slot, parts).double()                                # [N, parts]
    want_su, want_sq = ref @ S, ref.square() @ S                       # [M, parts]
    tol_su = 2 * (e @ S + 40 * U * (ref.abs() @ S))
    tol_sq = 2 * (((2 * ref.abs() + e) * e) @ S + 40 * U * want_sq)
    got = stats[:parts].double().permute(1, 0, 2)                      # [M, parts, 2]
    check(got[..., 0], want_su, tol_su, 0.0, f"{case['id']}: row sums per partial")
    check(got[..., 1], want_sq, tol_sq, 0.0, f"{case['id']}: row sums of squares per partial")
    return out, ref, e, plan


def _im2col64(x, cmode):
    """NHWC bf16 [B, H, W, C] -> fp64 [B * Ho * Wo, 9 C] in the packed weights' (ky, kx, c) order"""
    B, H, W, C = x.shape
    xin = x.double().permute(0, 3, 1, 2)
    if cmode == 2:
        xp, stride = F.pad(xin, (0, 1, 0, 1)), 2
    else:
        xp, stride = F.pad(xin, (1, 1, 1, 1)), (2 if cmode == 1 else 1)
    cols = F.unfold(xp, 3, stride=stride)                              # [B, C * 9, L], (c, ky, kx)
    L = cols.shape[-1]
    return cols.view(B, C, 9, L).permute(0, 3, 2, 1).reshape(B * L, 9 * C)


def _taps64(x, par):
    """NHWC bf16 [B, H, W, C] -> fp64 [B * H * W, 4 C]: the 2x2 source taps of output parity par = 2 py + px of the folded
    upsample conv, K ordered (ty, tx, c), source pixel (y + ty - 1 + py, x + tx - 1 + px), zero outside the image"""
    B, H, W, C = x.shape
    py, px = par >> 1, par & 1
    xp = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1))
    taps = [xp[:, :, py + ty:py + ty + H, px + tx:px + tx + W] for ty in (0, 1) for tx in (0, 1)]
    return torch.cat(taps, 1).permute(0, 2, 3, 1).reshape(B * H * W, 4 * C)


def run_conv(case):
    """vdb_conv3x3_bf16 as the GEMM im2col(x) W^T (+ bias, act, residual), bounded as a plain GEMM with K = 9 C (4 C for the
    folded upsample modes).  Modes 7..10 write one parity of a zero-filled [B, 2H, 2W, N] tensor: the other three parities
    must stay zero."""
    ops = _ops()
    B, H, W, C, N, cmode, act = case["B"], case["H"], case["W"], case["C"], case["N"], case["cmode"], case.get("act", 0)
    Ho, Wo = (H // 2, W // 2) if cmode in (1, 2) else (H, W)
    taps = 4 if cmode >= 3 else 9
    x = rnd(B, H, W, C, seed=1)
    w = rnd(N, taps * C, seed=2, scale=(taps * C) ** -0.5)
    rows = B * Ho * Wo
    b, bstride, _ = _bias(dict(case, rpb=Ho * Wo), rows, N, 3)
    r = rnd(B, Ho, Wo, N, seed=4) if case.get("resid") else None
    f32 = case.get("f32", False)
    full = torch.zeros(B, 2 * H, 2 * W, N, dtype=torch.bfloat16, device=DEV) if cmode >= 7 else None
    out = ops.conv3x3(x, w, bias=b, bias_bstride=bstride, resid=r, act=act, mode=cmode, bn=case["bn"], ksplit=case["ksplit"],
                      out=full, out_dtype=torch.float32 if f32 else torch.bfloat16)
    plan = ops.igemm_last_plan()
    if cmode >= 7:
        py, px = (cmode - 7) >> 1, (cmode - 7) & 1
        others = torch.ones(2 * H, 2 * W, dtype=torch.bool, device=DEV)
        others[py::2, px::2] = False
        assert torch.count_nonzero(full[:, others]) == 0, f"{case['id']}: a store left its parity"
        out = full[:, py::2, px::2, :].contiguous()
    xc = _taps64(x, (cmode - 3) % 4) if cmode >= 3 else _im2col64(x, cmode)
    pre = mm64(xc, w) + _bias_rows(b, bstride, Ho * Wo, rows)
    ref = act64(pre, act)
    atol = 1.25 * (4 * taps * C * U * rss64(xc, w) + 2 * U * pre.abs()) + 2.0 ** -20 * pre.abs()
    if r is not None:
        ref = ref + r.double().view(rows, N)
        atol = atol + 2.0 ** -20 * r.double().view(rows, N).abs()
    return out.view(rows, N), ref, atol, plan


RUN = {"gemm": run_gemm, "ln": run_ln, "stats": run_stats, "conv": run_conv}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_instantiation(case):
    out, ref, atol, plan = RUN[case["kind"]](case)
    check_plan(case, plan)
    check(out, ref, atol, 2.0 ** -16 if case.get("f32") else 2.0 ** -8, case["id"])

