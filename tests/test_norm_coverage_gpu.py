"""Every GroupNorm and LayerNorm kernel instantiation (elementwise.cu), and the state the single-launch GroupNorm carries from
one launch to the next, against an fp64 reference.

vdb_groupnorm_nhwc chooses between seven kernels: gn_bundle_kernel <2,512>, <6,512>, <12,512> and <11,1024> (clusters of
S = 1, 2, 4 or 8 CTAs), gn_fused_kernel <4> and <0> (one launch, a device-wide per-image arrival counter), and gn_stats_kernel
followed by gn_apply_kernel.  vdb_layernorm chooses between layernorm_rg_kernel <VPL, LPR> at eight channel counts and
layernorm_kernel <2,4>, <5,2>, <8,1>.  Each row of the tables below names the instantiation it targets; the test asserts the
plan the launcher reports (ops.norm_last_plan) and compares every output element with the fp64 restatement on the same bf16
input: F.group_norm (then SiLU) and F.layer_norm.  The dispatch depends on the SM count; the tables are laid out for the 132 SMs
of an H100 SXM (on another part the numerics still run, the plan assertions are skipped).  The inputs have groups / rows with
mean / std of 0, 8 and 64, channels of one group with different means, a constant group / row, and (VAE rows) |x| up to ~1e3.

Tolerance, per element (u = 2^-24, fp32 unit roundoff):
    |out - ref| <= 2^-8 |ref| + atol
  2^-8 |ref| is the bf16 rounding of the output (8 significant bits: at most 2^-8 / (1 + 2^-8) of the value, and measured
  elements reach 0.996 of that), so every margin sits in atol.  With x^ = (x - mean) rstd the normalised input:

  GroupNorm (all three paths).  Every path sums x and x^2 per group in fp32 and forms var = E[x^2] - mean^2, so the variance
  loses (E[x^2] / (var + eps)) times the relative error of the sums; rstd = rsqrt(var + eps) halves that and adds rsqrtf's
  2 ulps.  With the sums' relative error at a few u (the bundle kernel's fold order, emulated in fp32, gives 8e-4 on the variance
  at mean / std = 128, i.e. 0.8 u E[x^2] / var):
      eps_r = 2^-22 (1 + E[x^2] / (var + eps))
      atol  = |gamma_c| |x^| eps_r + 2^-20 (|beta_c| + |mean_g rstd_g gamma_c|)
  the second term covers the mean's rounding (seen through rstd gamma) and the fp32 x * scale + shift with
  scale = rstd gamma, shift = beta - mean scale.  SiLU (x/2 (1 + tanh.approx(x/2)), tanh.approx: 2^-11 relative) adds
  2^-12 |y| of the pre-activation y, and the activation's slope (< 1.1) multiplies atol.  A constant group (var = 0) has x^ = 0:
  its output is beta_c up to the mean's rounding times rstd = 1/sqrt(eps).

  LayerNorm (both kernels) is two-pass: mean = sum(x) / C, then var = sum((x - mean)^2) / C.  A lane sums its V values
  sequentially and the row's lanes fold in a butterfly, depth D = 8 VPL + log2(LPR) (row-group) or 8 MAXV + 5 (warp per row);
  the sums' first-order error is D u times the sum of |terms|.  var has no cancellation, so
      atol = |gamma_c| |x^| (D / 2 + 4) u + |gamma_c| rstd (D + 1) u mean|x| + 4 u |beta_c|
  (rstd from var and rsqrtf; the mean's error through rstd gamma; the fp32 affine).

  affine_act_rows: y = x gamma + beta in fp32, atol = 4 u (|x gamma| + |beta|), SiLU as above.

The cosine >= 0.999 check of test_kernels_gpu is kept as a second guard.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
BF16 = torch.bfloat16
SMS_LAYOUT = 132           # the SM count the tables below were laid out for (H100 SXM)
REACHED = set()            # plans reached by the case tests (test_every_instantiation_reached)
RAN = set()


def _ops():
    from vdb200 import ops
    return ops


def _layout_ok():
    return _ops().lib.vdb_num_sms() == SMS_LAYOUT


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def plan_key(plan):
    f = plan["family"]
    if f == "gn_bundle":
        return (f, plan["t0"], plan["t1"], plan["S"])
    if f == "gn_fused":
        return (f, plan["t0"])
    if f == "gn_stats_apply":
        return (f,)
    return (f, plan["t0"], plan["t1"])


def check(out, ref, atol, what, rtol=2.0 ** -8):
    out = out.double()
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs()
    lim = rtol * ref.abs() + atol
    bad = err > lim
    if bad.any():
        i = int((err - lim).argmax())
        idx = [int(j) for j in torch.unravel_index(torch.tensor(i), err.shape)]
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of tolerance; worst at {idx}: "
                             f"out {out.flatten()[i].item():.6g} ref {ref.flatten()[i].item():.6g} limit {lim.flatten()[i].item():.3g}")
    cos = F.cosine_similarity(out.flatten(), ref.flatten(), dim=0).item()
    assert cos >= 0.999, f"{what}: cosine {cos:.6f}"


# ---------------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------------
def _gn(cid, B, HW, C1, C2=0, act=1, eps=1e-5, want=None, scale=1.0):
    return dict(id=cid, B=B, HW=HW, C1=C1, C2=C2, act=act, eps=eps, want=want, scale=scale)


def bundle(nv, threads, G, S):
    return dict(family="gn_bundle", t0=nv, t1=threads, G=G, S=S)


def fused(nv):
    return dict(family="gn_fused", t0=nv)


STATS = dict(family="gn_stats_apply")

GN_CASES = [
    # gn_bundle_kernel<2, 512>: HW down to 1 (the 0-D diffuser's FCBlock: HW = sdim), G = 1 / 4 / 2, S = 1 .. 8
    _gn("b2-s1-hw1-c1280", 8, 1, 1280, want=bundle(2, 512, 1, 1)),
    _gn("b2-s1-hw1-c320-g4", 4, 1, 320, act=0, eps=1e-6, want=bundle(2, 512, 4, 1)),
    _gn("b2-s1-hw3-c640-g2", 2, 3, 640, want=bundle(2, 512, 2, 1)),
    _gn("b2-s2-g2-concat", 1, 400, 256, 128, eps=1e-6, want=bundle(2, 512, 2, 2)),           # boundary inside bundle 10
    _gn("b2-s4-g4-concat", 1, 144, 640, 320, act=0, want=bundle(2, 512, 4, 4)),              # boundary inside bundle 5
    _gn("b2-s8-partial", 1, 4999, 256, want=bundle(2, 512, 1, 8)),                           # last rank: 624 of 625 pixels
    _gn("b2-s8-g4", 2, 1024, 320, eps=1e-6, want=bundle(2, 512, 4, 8)),
    # gn_bundle_kernel<6, 512>
    _gn("b6-s1", 8, 577, 512, want=bundle(6, 512, 1, 1)),
    _gn("b6-s2-partial", 3, 2501, 256, act=0, eps=1e-6, want=bundle(6, 512, 1, 2)),
    _gn("b6-s4-g2-concat", 3, 1500, 200, 184, want=bundle(6, 512, 2, 4)),
    _gn("b6-s4-g4", 8, 1500, 192, eps=1e-6, want=bundle(6, 512, 4, 4)),
    _gn("b6-s8", 1, 9000, 256, act=0, want=bundle(6, 512, 1, 8)),
    # gn_bundle_kernel<11, 1024> (pixels staged in shared memory)
    _gn("b11-s1", 2, 9001, 256, want=bundle(11, 1024, 1, 1)),
    _gn("b11-s1-g2", 2, 8192, 128, act=0, eps=1e-6, want=bundle(11, 1024, 2, 1)),
    _gn("b11-s2", 1, 16384, 256, want=bundle(11, 1024, 1, 2)),
    _gn("b11-s2-g4", 4, 4096, 192, eps=1e-6, want=bundle(11, 1024, 4, 2)),
    _gn("b11-s4-g4", 2, 8192, 192, act=0, want=bundle(11, 1024, 4, 4)),
    _gn("b11-s4-g2-concat", 2, 8192, 200, 184, eps=1e-6, want=bundle(11, 1024, 2, 4)),
    _gn("b11-s8-concat", 1, 16384, 648, 632, want=bundle(11, 1024, 1, 8)),                   # boundary inside bundle 16
    _gn("b11-s8-g2", 1, 16384, 384, act=0, eps=1e-6, want=bundle(11, 1024, 2, 8)),
    # gn_bundle_kernel<12, 512>: only ever at S = 8
    _gn("b12-s8-vae", 8, 16384, 512, eps=1e-6, want=bundle(12, 512, 1, 8), scale=8.0),
    _gn("b12-s8-concat", 1, 5000, 640, 640, act=0, want=bundle(12, 512, 1, 8)),
    _gn("b12-s8-g4-partial", 1, 8191, 192, eps=1e-6, want=bundle(12, 512, 4, 8)),
    # gn_fused_kernel<4>: fewer than 4 channels per group (no bundle), or cpg = 5 (no 16-byte bundle with G <= 4)
    _gn("f4-c32", 4, 1024, 32, want=fused(4)),
    _gn("f4-c64", 2, 4096, 64, act=0, eps=1e-6, want=fused(4)),
    _gn("f4-c96-partial", 3, 700, 96, eps=1e-6, want=fused(4)),
    _gn("f4-c160-concat", 8, 256, 96, 64, act=0, want=fused(4)),
    # gn_fused_kernel<0>: the VAE decoder's GroupNorms at 256^2 and 512^2 for 4 images, VAE-like magnitudes
    _gn("f0-vae-65536x512", 4, 65536, 512, eps=1e-6, want=fused(0), scale=8.0),
    _gn("f0-vae-65536x256", 4, 65536, 256, act=0, eps=1e-6, want=fused(0), scale=8.0),
    _gn("f0-vae-262144x256", 4, 262144, 256, eps=1e-6, want=fused(0), scale=8.0),
    _gn("f0-vae-262144x128", 4, 262144, 128, eps=1e-6, want=fused(0), scale=8.0),
    _gn("f0-concat", 4, 65536, 256, 128, eps=1e-5, want=fused(0)),
    _gn("f0-c32", 4, 40000, 32, act=0, want=fused(0)),
    # gn_stats_kernel + gn_apply_kernel: C > 3072, or more images than resident single-launch CTAs
    _gn("sa-c3104-concat", 2, 3000, 1552, 1552, want=STATS),
    _gn("sa-b300", 300, 256, 64, act=0, eps=1e-6, want=STATS),
    _gn("sa-b300-hw1000", 300, 1000, 64, eps=1e-5, want=STATS, scale=8.0),
]

CONST_GROUP = 3


def gn_input(B, HW, C, seed, scale=1.0):
    """[B, HW, C] bf16: group g of image b has std s in [0.5, 2] scale and mean (0, 8, 64)[g % 3] s (random sign), its channels
    carry extra means in [-s/2, s/2]; group CONST_GROUP is constant (2.5 scale)"""
    g = _gen(seed)
    cpg = C // 32
    sig = (torch.rand(B, 32, generator=g, device=DEV) * 1.5 + 0.5) * scale
    ratio = torch.tensor([0.0, 8.0, 64.0], device=DEV).repeat(11)[:32]
    sign = torch.where(torch.rand(B, 32, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    sig_c = sig.repeat_interleave(cpg, 1)
    mean_c = (ratio * sig * sign).repeat_interleave(cpg, 1) + (torch.rand(B, C, generator=g, device=DEV) - 0.5) * sig_c
    x = torch.randn(B, HW, C, generator=g, device=DEV)
    x.mul_(sig_c[:, None, :]).add_(mean_c[:, None, :])
    x[:, :, CONST_GROUP * cpg:(CONST_GROUP + 1) * cpg] = 2.5 * scale
    return x.to(BF16)


def gn_params(C, seed):
    g = _gen(seed)
    return torch.randn(C, generator=g, device=DEV), torch.randn(C, generator=g, device=DEV)


def gn_split(x, C1):
    if C1 == x.shape[-1]:
        return x, None
    return x[..., :C1].contiguous(), x[..., C1:].contiguous()


def gn_call(x1, x2, gamma, beta, eps, act, scratch, out):
    """vdb_groupnorm_nhwc on an explicit scratch buffer (ops.groupnorm keeps one per stream)"""
    ops = _ops()
    B, C1 = x1.shape[0], x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    HW = x1.numel() // (B * C1)
    ops.check(ops.lib.vdb_groupnorm_nhwc(ops._ptr(x1), C1, ops._ptr(x2), C2, B, HW, 32, ops._ptr(gamma), ops._ptr(beta),
                                         float(eps), int(act), ops._ptr(scratch), ops._ptr(out), ops._stream()), "groupnorm_nhwc")
    return out


def gn_scratch(shapes):
    ops = _ops()
    n = max(ops.lib.vdb_groupnorm_scratch_floats(B, HW) for B, HW in shapes)
    return torch.zeros(n, dtype=torch.float32, device=DEV)


def gn_check(out, x, gamma, beta, eps, act, what):
    """every element against F.group_norm in fp64 (then SiLU), one image at a time"""
    B, HW, C = x.shape
    cpg = C // 32
    gam, bet = gamma.double(), beta.double()
    for b in range(B):
        xb = x[b].double()                                                        # [HW, C]
        y = F.group_norm(xb.t().unsqueeze(0), 32, gam, bet, eps)[0].t()
        xg = xb.view(HW, 32, cpg)
        mean = xg.mean((0, 2))
        var = (xg - mean[None, :, None]).square().mean((0, 2))
        ex2 = xg.square().mean((0, 2))
        rstd = (var + eps).rsqrt()
        eps_r = 2.0 ** -22 * (1 + ex2 / (var + eps))
        mean_c, rstd_c, eps_c = (t.repeat_interleave(cpg) for t in (mean, rstd, eps_r))
        xhat = (xb - mean_c) * rstd_c
        atol = gam.abs() * xhat.abs() * eps_c + 2.0 ** -20 * (bet.abs() + (mean_c * rstd_c * gam).abs())
        del xg, xhat
        if act:
            ref = F.silu(y)
            atol = 1.1 * atol + 2.0 ** -12 * y.abs()
        else:
            ref = y
        check(out[b].reshape(HW, C), ref, atol, f"{what} image {b}")


def check_gn_plan(case, plan):
    want = case["want"]
    if want["family"] == "gn_bundle":
        C = case["C1"] + case["C2"]
        assert plan["grid_x"] * plan["G"] == 32 and plan["grid_y"] == plan["S"] and plan["grid_z"] == case["B"], plan
        assert (C // 32) * plan["G"] % 8 == 0, plan
    else:
        assert plan["grid_y"] == case["B"] and plan["grid_x"] == plan["nsplit"], plan
    got = {k: plan[k] for k in want}
    assert got == want, f"{case['id']}: launched {plan}, case expects {want}"


@pytest.mark.parametrize("case", GN_CASES, ids=[c["id"] for c in GN_CASES])
def test_groupnorm_case(case):
    ops = _ops()
    B, HW, C1, C2 = case["B"], case["HW"], case["C1"], case["C2"]
    C = C1 + C2
    x = gn_input(B, HW, C, seed=B * 7 + HW + C, scale=case["scale"])
    gamma, beta = gn_params(C, seed=C + 1)
    x1, x2 = gn_split(x, C1)
    scratch = gn_scratch([(B, HW)])
    out = gn_call(x1, x2, gamma, beta, case["eps"], case["act"], scratch, torch.empty(B, HW, C, dtype=BF16, device=DEV))
    plan = ops.norm_last_plan()
    REACHED.add(plan_key(plan))
    RAN.add(case["id"])
    if _layout_ok():
        check_gn_plan(case, plan)
    again = gn_call(x1, x2, gamma, beta, case["eps"], case["act"], scratch, torch.empty_like(out))
    assert torch.equal(out, again), f"{case['id']}: not run-to-run deterministic"
    assert not scratch[:2048].view(torch.int32).any(), f"{case['id']}: counters left armed"
    gn_check(out, x, gamma, beta, case["eps"], case["act"], case["id"])


# state carried between launches: the single-launch kernel's arrive / depart counters and the statistics kernel's counters
# share the front of the scratch buffer; the partial sums and statistics behind them are rewritten by every launch
SEQUENCE = [
    _gn("f0", 4, 65536, 256, want=fused(0)),
    _gn("bundle", 2, 1024, 320, want=bundle(2, 512, 4, 8)),
    _gn("f4", 8, 1024, 64, act=0, eps=1e-6, want=fused(4)),
    _gn("stats", 300, 256, 64, want=STATS),
]


def _seq_inputs(case, k):
    C = case["C1"] + case["C2"]
    x = gn_input(case["B"], case["HW"], C, seed=100 + k)
    g, b = gn_params(C, seed=200 + k)
    return x, g, b


def test_groupnorm_state_across_launches():
    """fused<0> (B 4) -> bundle -> fused<4> (B 8) -> stats + apply (B 300) -> fused<0> again on ONE scratch buffer: each output
    bitwise equal to a run on a fresh zeroed scratch, and within the fp64 bound"""
    ops = _ops()
    if not _layout_ok():
        pytest.skip(f"sequence laid out for {SMS_LAYOUT} SMs")
    seq = SEQUENCE + [SEQUENCE[0]]
    inputs = [_seq_inputs(c, k % len(SEQUENCE)) for k, c in enumerate(seq)]
    shared = gn_scratch([(c["B"], c["HW"]) for c in seq])
    for k, (case, (x, g, b)) in enumerate(zip(seq, inputs)):
        x1, x2 = gn_split(x, case["C1"])
        out = gn_call(x1, x2, g, b, case["eps"], case["act"], shared, torch.empty_like(x))
        plan = ops.norm_last_plan()
        check_gn_plan(case, plan)
        fresh = gn_call(x1, x2, g, b, case["eps"], case["act"], gn_scratch([(case["B"], case["HW"])]), torch.empty_like(x))
        assert torch.equal(out, fresh), f"launch {k} ({case['id']}) on the shared scratch differs from a fresh run"
        gn_check(out, x, g, b, case["eps"], case["act"], f"launch {k} ({case['id']})")
    assert not shared[:2048].view(torch.int32).any(), "counters left armed"


def test_groupnorm_fused_graph_replay():
    """two fused<0> launches captured in one CUDA graph, replayed three times: bitwise the eager result each time"""
    ops = _ops()
    case = SEQUENCE[0]
    xa, ga, ba = _seq_inputs(case, 0)
    xb, gb, bb = _seq_inputs(case, 5)
    scratch = gn_scratch([(case["B"], case["HW"])])
    ya, yb = torch.empty_like(xa), torch.empty_like(xb)
    gn_call(xa, None, ga, ba, 1e-5, 1, scratch, ya)
    assert ops.norm_last_plan()["family"] == "gn_fused" or not _layout_ok()
    gn_call(xb, None, gb, bb, 1e-6, 0, scratch, yb)
    ea, eb = ya.clone(), yb.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gn_call(xa, None, ga, ba, 1e-5, 1, scratch, ya)
        gn_call(xb, None, gb, bb, 1e-6, 0, scratch, yb)
    for _ in range(3):
        ya.zero_(); yb.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ya, ea) and torch.equal(yb, eb), "graph replay differs from eager"
    assert not scratch[:2048].view(torch.int32).any(), "counters left armed"


# ---------------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------------
LN_INST = [  # (C, family, T0, T1)
    (64, "ln_rg", 1, 8), (128, "ln_rg", 2, 8), (256, "ln_rg", 4, 8), (320, "ln_rg", 5, 8), (640, "ln_rg", 5, 16),
    (768, "ln_rg", 3, 32), (1024, "ln_rg", 4, 32), (1280, "ln_rg", 5, 32),
    (96, "ln_warp", 2, 4), (384, "ln_warp", 2, 4), (1000 // 8 * 8, "ln_warp", 5, 2), (1536, "ln_warp", 8, 1), (2048, "ln_warp", 8, 1),
]


def _rows_per_step(family, t1):
    return 32 // t1 if family == "ln_rg" else t1          # rows a warp takes per step: 32 / LPR, or R


def _ln_rows(family, t1):
    """1, fewer than one warp step, a partial last step, and more than any grid can cover in one step (<= 8 CTAs of 8 warps
    per SM), so the persistent walk wraps"""
    rps = _rows_per_step(family, t1)
    rows = {1, max(1, rps - 1), 5 * rps + 1 if rps > 1 else 77, 8 * 8 * SMS_LAYOUT * rps + 37}
    return sorted(rows)


LN_CASES = [dict(id=f"{fam}-c{C}-r{r}", C=C, rows=r, family=fam, t0=t0, t1=t1, wrap=r > 8 * 8 * SMS_LAYOUT * _rows_per_step(fam, t1),
                 eps=1e-5 if C % 3 else 1e-6)
            for C, fam, t0, t1 in LN_INST for r in _ln_rows(fam, t1)]


def ln_input(rows, C, seed):
    """row i: std s in [0.5, 2], mean (64, 0, 8, 1)[i % 4] s (random sign); row 5 constant"""
    g = _gen(seed)
    sd = torch.rand(rows, 1, generator=g, device=DEV) * 1.5 + 0.5
    ratio = torch.tensor([64.0, 0.0, 8.0, 1.0], device=DEV)[torch.arange(rows, device=DEV) % 4][:, None]
    sign = torch.where(torch.rand(rows, 1, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    x = torch.randn(rows, C, generator=g, device=DEV) * sd + ratio * sd * sign
    if rows > 5:
        x[5] = -2.5
    return x.to(BF16)


def ln_check(out, x, gamma, beta, eps, depth, what):
    xd = x.double()
    gam, bet = gamma.double(), beta.double()
    ref = F.layer_norm(xd, (x.shape[1],), gam, bet, eps)
    mean = xd.mean(1, keepdim=True)
    rstd = ((xd - mean).square().mean(1, keepdim=True) + eps).rsqrt()
    xhat = (xd - mean) * rstd
    atol = (gam.abs() * xhat.abs() * (depth / 2 + 4) * U + gam.abs() * rstd * (depth + 1) * U * xd.abs().mean(1, keepdim=True)
            + 4 * U * bet.abs())
    check(out, ref, atol, what)


@pytest.mark.parametrize("case", LN_CASES, ids=[c["id"] for c in LN_CASES])
def test_layernorm_case(case):
    ops = _ops()
    C, rows = case["C"], case["rows"]
    x = ln_input(rows, C, seed=rows + C)
    gamma, beta = gn_params(C, seed=C + 2)
    out = ops.layernorm(x, gamma, beta, case["eps"])
    plan = ops.norm_last_plan()
    REACHED.add(plan_key(plan))
    RAN.add(case["id"])
    want = {k: case[k] for k in ("family", "t0", "t1")}
    assert {k: plan[k] for k in want} == want, f"{case['id']}: launched {plan}, case expects {want}"
    if case["wrap"] and _layout_ok():
        assert plan["grid_x"] * 8 * _rows_per_step(case["family"], case["t1"]) < rows, f"{case['id']}: the walk does not wrap ({plan})"
    assert torch.equal(out, ops.layernorm(x, gamma, beta, case["eps"])), f"{case['id']}: not run-to-run deterministic"
    depth = 8 * case["t0"] + (int(math.log2(case["t1"])) if case["family"] == "ln_rg" else 5)
    ln_check(out, x, gamma, beta, case["eps"], depth, case["id"])


# ---------------------------------------------------------------------------------------------------------------------------
# affine_act_rows (FCBlock's per-position GroupNorm affine)
# ---------------------------------------------------------------------------------------------------------------------------
AFFINE_CASES = [(rows, n, act) for rows, n in ((1, 8), (3, 48), (1000, 8), (77, 5120), (70001, 64)) for act in (0, 1)]


@pytest.mark.parametrize("rows,n,act", AFFINE_CASES)
def test_affine_act_rows(rows, n, act):
    """y = act(x gamma + beta) per element; 70001 x 64 is more 16-byte vectors than the grid covers in one pass"""
    ops = _ops()
    g = _gen(rows * 31 + n)
    x = (torch.randn(rows, n, generator=g, device=DEV) * 4).to(BF16)
    gamma = torch.randn(n, generator=g, device=DEV) * 2
    beta = torch.randn(n, generator=g, device=DEV)
    out = ops.affine_silu_rows(x, gamma, beta, act=act)
    y = x.double() * gamma.double() + beta.double()
    atol = 4 * U * ((x.double() * gamma.double()).abs() + beta.double().abs())
    if act:
        ref, atol = F.silu(y), 1.1 * atol + 2.0 ** -12 * y.abs()
    else:
        ref = y
    check(out, ref, atol, f"affine_act_rows {rows}x{n} act {act}")
    assert torch.equal(out, ops.affine_silu_rows(x, gamma, beta, act=act))


# ---------------------------------------------------------------------------------------------------------------------------
def expected_instantiations():
    """every kernel instantiation the dispatch can launch, at every cluster size it can give it"""
    want = {("gn_bundle", nv, th, s) for nv, th in ((2, 512), (6, 512), (11, 1024)) for s in (1, 2, 4, 8)}
    want |= {("gn_bundle", 12, 512, 8), ("gn_fused", 4), ("gn_fused", 0), ("gn_stats_apply",)}
    want |= {(fam, t0, t1) for _, fam, t0, t1 in LN_INST}
    return want


def test_every_instantiation_reached():
    """the case tests above reached exactly the full list of instantiations: a dispatch change that drops one (or adds one
    nothing here covers) fails here"""
    if not _layout_ok():
        pytest.skip(f"tables laid out for {SMS_LAYOUT} SMs")
    ids = {c["id"] for c in GN_CASES} | {c["id"] for c in LN_CASES}
    if RAN != ids:
        pytest.skip("runs after the whole case table")
    want = expected_instantiations()
    assert len(want) == 16 + 11
    assert REACHED == want, f"missing {sorted(want - REACHED)}, unexpected {sorted(REACHED - want)}"
