"""The text decoder's token-step kernels (textdec.cu) element by element against fp64, at every K-split, grid-stride count, row
count, LayerNorm and epilogue path of the GEMV, and the KV-cache step, the embedding and the sampler's bookkeeping.

vdb_textdec_gemv splits K over ks in {1, 2, 4, 8} warps of a CTA: ks doubles while tiles * ks < 16 * SMs (tiles = N / 8 rounded
up) and K / 32 stays divisible by 2 ks, and min(tiles / (8 / ks), 2 * SMs) CTAs walk the tiles in a grid-stride loop.  gemv_plan
restates that rule; each case names the ks and the number of loop iterations it reaches on the 132 SMs of an H100 SXM (on
another part the numerics still run, the reach assertions are skipped).  Each case runs five launches on the same x:

  staged operand   W = the bf16 identity (N = K), no bias.  Each output is 1 * x~ plus exact zeros, so it is the kernel's bf16
                   operand x~ bit for bit.  Without LayerNorm x~ must equal x.to(bfloat16).  With it, x~ is the fp32 two-pass
                   LayerNorm rounded to bf16; with y the fp64 F.layer_norm and e the fp32 error bound below, x~ must lie in
                   [bf16(y - e), bf16(y + e)] (rounding is monotone): bf16(y) itself except where y is within e of a rounding
                   midpoint.  The prologue is the same code in every CTA whatever N and ks are, so this x~ is also the operand
                   of the dense launches.
                   LayerNorm bound (test_norm_coverage_gpu's two-pass derivation, u = 2^-24): a lane sums K / 32 values in
                   order and the warp folds in a 5-level butterfly, depth D = K / 32 + 5, so
                       e = |g| |x^| (D / 2 + 4) u + |g| rstd (D + 1) u mean|x| + 4 u |b|
                   A constant row has x^ = 0 and rstd = 1 / sqrt(eps): its output is b up to the mean's rounding times rstd,
                   which the second term covers.
  dense, act NONE  ref = x~ . W^T + bias in fp64.  bf16 x bf16 products are exact in fp32, so only the accumulation errs: at
                   most 2^-22 of the running magnitude per mma step (the tensor cores truncate their fp32 sums).  Each of the
                   ks warps of a tile accumulates its own K / ks slice, a chain of K / (16 ks) steps; then ks - 1 partial sums
                   in shared memory and the bias add, each u:
                       |out - ref| <= (K / (16 ks) + ks + 2) 2^-22 (sum_k |w_nk x~_k| + |b_n|)
                   The bound is worst case; random-sign dot products land 1e-3 to 1e-1 of it.
  act GELU_TANH    the same launch configuration, so the pre-activation is bit for bit the NONE output v.  ref = optimus_gpt2's
                   0.5 v (1 + tanh(sqrt(2 / pi) (v + 0.044715 v^3))) in fp64.  The fp32 argument a has all terms of one sign:
                   |da| <= 6 u |a|; tanhf is within 2 ulps, so |dt| <= 6 u max(a sech^2 a) + 2^-22 < 7 u; 1 + t and the last
                   product add u each: |dg| <= 0.5 |v| (7 u + 2 u) + u |g| < 2^-21.4 |v|.  Tolerance 2^-20 |v|.
  act TANH         ref = tanh(v): tanhf's documented 2 ulps, 2^-22 |ref|.
  accumulate       out pre-filled with o0, act NONE: out must equal the fp32 o0 + v bitwise (the decoder's residual adds).  An
                   activation with accumulate is left out: nvcc may fuse its last product into the add, and no caller uses it.
Rows of the out slice outside [0, R) and columns >= N of a wider out hold a sentinel that must survive every launch, and the
columns of x and W outside the slice the kernel is given are NaN.

vdb_textdec_attention, one warp per (row, head): fp64 softmax over [latent slice, kc[0 .. s-1], k_new] * scale applied to
[latent, vc[0 .. s-1], v_new].  The error of the weight p_j of key j, relative:
  - the score: two lane products (one fused) and a 5-level butterfly, E_j = 7 u scale sum_d |q_d k_jd| (scale is a power of 2);
  - __expf(sc_j - m_j), m_j the running maximum: the documented 2 + 1.173 |x| ulps (<= 2^-23 each) plus the argument's
    rounding u |x|: x(a) = 2^-23 (2 + 1.173 a) + u a at a = m_j - sc_j;
  - each later rescale corr_i = __expf(m_{i-1} - m_i) (exact 1 when the maximum stays) multiplies l and acc alike, so it
    scales every earlier weight against the later ones by x(m_i - m_{i-1}): S_j = sum_{i > j} x(m_i - m_{i-1}).
A common relative error of all weights cancels in acc / l, so to first order |out - ref| <= sum_j p_j d_j |v_j - ref| with
d_j = E_j + x(m_j - sc_j) + S_j.  The n = s + 2 steps of the recurrence round l once (u |l|) and acc twice (u sum p |v|) each,
and the final division once:
    |out - ref| <= sum_j p_j d_j |v_j - ref| + 2 n u sum_j p_j |v_j| + (n + 1) u |ref|
q is scaled so the scores span about +-40 (the rescale's corr is far from 1), and a third of the (row, head) pairs have their
maximum at the latent key, a third at the new key.

vdb_textdec_embed is exact: (wte[tok] + wpe[pos]) + emb in fp32, bitwise, with the token clamped into [0, V - 1] and the position
s + pos_offset clamped to P - 1.  vdb_textdec_sample is checked for its bookkeeping only (finished rows, <eos>, the forced last
<eos>, teacher forcing, strided logits and the record); its draw is covered by test_text_decode_gpu and test_text_filter_gpu.
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
SENTINEL = -7777.0
REACHED = set()            # (ks, grid-stride iterations) of the GEMV cases run (test_every_path_reached)
RAN = set()


def _ops():
    from vdb200 import ops
    return ops


def _num_sms():
    return _ops().lib.vdb_num_sms()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def gemv_plan(K, N, sms):
    """(ks, grid-stride iterations of the busiest CTA) that vdb_textdec_gemv launches"""
    tiles, want, chunks = (N + 7) // 8, sms * 2 * 8, K // 32
    ks = 1
    while ks < 8 and tiles * ks < want and chunks % (2 * ks) == 0:
        ks *= 2
    slots = 8 // ks
    blocks = min(-(-tiles // slots), 2 * sms)
    return ks, -(-tiles // (blocks * slots))


def worst(ratio):
    return ratio.max().item() if ratio.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_textdec_gemv
# ---------------------------------------------------------------------------------------------------------------------------
def _gv(cid, R, K, N, ks, iters, ln=True, bias=True, padx=0, padw=0, pado=0):
    return dict(id=cid, R=R, K=K, N=N, want=(ks, iters), ln=ln, bias=bias, padx=padx, padw=padw, pado=pado)


GEMV_CASES = [
    # the decoder's own launches
    _gv("lm_head-ln_f", 16, 768, 50260, 1, 3, bias=False, pado=4),             # N % 8 = 4: the tail tile's nrow clamp
    _gv("linear", 4, 768, 9216, 2, 2, ln=False, bias=False, padx=24),
    _gv("c_attn-ln_1", 16, 768, 2304, 8, 2, padw=8),                          # the second iteration: 24 of 264 CTAs busy
    _gv("c_fc-ln_2", 1, 768, 3072, 8, 2, pado=3),
    _gv("mlp.c_proj", 8, 3072, 768, 8, 1, ln=False, padx=5),                  # K = 3072: the largest shared operand
    # the other splits, row counts and edges
    _gv("r9-ks4", 9, 768, 6000, 4, 2, padx=7, padw=16, pado=1),
    _gv("k32-n7", 3, 32, 7, 1, 1, pado=9),                                    # one chunk, one partial tile
    _gv("k64-n1", 16, 64, 1, 2, 1, ln=False),
    _gv("k128-n100-nobias", 12, 128, 100, 4, 1, bias=False, padx=3, padw=8, pado=28),
    _gv("k96-unpadded", 5, 96, 520, 1, 1, padx=32, padw=24, pado=8),           # K % 64 == 32: the row stride is not padded
]
CONST = 7.0 / 3.0          # the constant row: its fp32 sums round, so the kernel's mean is not exactly CONST


def gemv_x(R, K, pad, seed):
    """fp32 [R, K] as a column slice of a [R, K + pad] buffer whose other columns are NaN.  Row i has std s in [0.5, 1.5] and
    mean (0, 8, 64)[i % 3] s of random sign (|x| up to ~1e2); the last row of R >= 3 is constant."""
    g = _gen(seed)
    sd = torch.rand(R, 1, generator=g, device=DEV) + 0.5
    ratio = torch.tensor([0.0, 8.0, 64.0], device=DEV)[torch.arange(R, device=DEV) % 3][:, None]
    sign = torch.where(torch.rand(R, 1, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    x = torch.randn(R, K, generator=g, device=DEV) * sd + ratio * sd * sign
    if R >= 3:
        x[R - 1] = CONST
    buf = torch.full((R, K + pad), float("nan"), device=DEV)
    off = pad // 2
    buf[:, off:off + K] = x
    return buf[:, off:off + K]


def gemv_w(N, K, pad, seed):
    """bf16 [N, K] (scale K^-1/2) as the columns 8.. of a NaN-padded [N, K + pad] buffer when pad > 0 (16-byte aligned)"""
    g = _gen(seed)
    w = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).to(BF16)
    if not pad:
        return w
    buf = torch.full((N, K + pad), float("nan"), dtype=BF16, device=DEV)
    buf[:, 8:8 + K] = w
    return buf[:, 8:8 + K]


def out_buffer(R, N, pad, fill=None):
    """[R + 2, N + pad] fp32 of SENTINEL; returns (buffer, the [R, N] slice at row 1), the slice set to fill when given"""
    buf = torch.full((R + 2, N + pad), SENTINEL, device=DEV)
    out = buf[1:R + 1, :N]
    if fill is not None:
        out.copy_(fill)
    return buf, out


def check_sentinel(buf, R, N, what):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[1:R + 1, :N] = False
    assert (buf[mask] == SENTINEL).all(), f"{what}: wrote outside out[0:{R}, 0:{N}]"


def run_gemv(x, w, R, N, pado, what, **kw):
    """one vdb_textdec_gemv into a sentinel-framed out; returns the [R, N] result"""
    fill = kw.pop("fill", None)
    buf, out = out_buffer(R, N, pado, fill)
    _ops().textdec_gemv(x, w, out, **kw)
    check_sentinel(buf, R, N, what)
    return out.clone()


def ln_bound(x, gamma, beta, eps):
    """the fp32 two-pass LayerNorm error bound e (module docstring), fp64 [R, K]"""
    K = x.shape[1]
    depth = K // 32 + 5
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    rstd = ((xd - mean).square().mean(1, keepdim=True) + eps).rsqrt()
    xhat = (xd - mean) * rstd
    gam, bet = gamma.double().abs(), beta.double().abs()
    return gam * xhat.abs() * (depth / 2 + 4) * U + gam * rstd * (depth + 1) * U * xd.abs().mean(1, keepdim=True) + 4 * U * bet


def check_staged(xs, x, ln, what):
    """xs: the identity run's output, the kernel's bf16 operand as fp32"""
    assert torch.isfinite(xs).all(), f"{what}: non-finite staged operand"
    assert torch.equal(xs, xs.to(BF16).float()), f"{what}: the identity product is not a bf16 value"
    if ln is None:
        assert torch.equal(xs, x.to(BF16).float()), f"{what}: staged operand != x.to(bfloat16)"
        return 0
    gamma, beta, eps = ln
    y = F.layer_norm(x.double(), (x.shape[1],), gamma.double(), beta.double(), eps)
    e = ln_bound(x, gamma, beta, eps)
    lo, hi = (y - e).to(BF16).double(), (y + e).to(BF16).double()
    xd = xs.double()
    bad = (xd < lo) | (xd > hi)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} staged LayerNorm elements outside [bf16(y - e), bf16(y + e)]; first at "
                             f"{divmod(i, x.shape[1])}: got {xd.flatten()[i].item():.8g}, fp64 {y.flatten()[i].item():.8g}, "
                             f"e {e.flatten()[i].item():.3g}")
    return int((xd != y.to(BF16).double()).sum())     # elements within e of a midpoint that rounded the other way


@pytest.mark.parametrize("case", GEMV_CASES, ids=[c["id"] for c in GEMV_CASES])
def test_gemv_case(case):
    ops = _ops()
    R, K, N = case["R"], case["K"], case["N"]
    plan = gemv_plan(K, N, _num_sms())
    if _num_sms() == SMS_LAYOUT:
        assert plan == case["want"], f"{case['id']}: the split rule gives (ks, iterations) {plan}, the case expects {case['want']}"
    ks = plan[0]
    seed = R * 131 + K * 7 + N
    x = gemv_x(R, K, case["padx"], seed)
    g = _gen(seed + 1)
    ln = None
    if case["ln"]:
        ln = (torch.randn(K, generator=g, device=DEV), torch.randn(K, generator=g, device=DEV), 1e-5)
    bias = torch.randn(N, generator=g, device=DEV) * 0.5 if case["bias"] else None
    w = gemv_w(N, K, case["padw"], seed + 2)
    pado = case["pado"]
    cid = case["id"]

    # the staged operand, through the identity
    xs = run_gemv(x, torch.eye(K, dtype=BF16, device=DEV), R, K, pado, f"{cid} identity", ln=ln)
    flips = check_staged(xs, x, ln, cid)

    # the dense product
    v = run_gemv(x, w, R, N, pado, f"{cid} dense", bias=bias, ln=ln)
    assert torch.isfinite(v).all(), f"{cid}: non-finite output"
    wd = w.double()
    ref = xs.double() @ wd.t()
    mag = xs.double().abs() @ wd.abs().t()
    if bias is not None:
        ref += bias.double()
        mag += bias.double().abs()
    bound = (K / (16 * ks) + ks + 2) * 2.0 ** -22 * mag
    r_dense = (v.double() - ref).abs() / bound
    assert worst(r_dense) <= 1.0, f"{cid}: dense err/bound {worst(r_dense):.3g} at {divmod(int(r_dense.argmax()), N)}"
    assert torch.equal(v, run_gemv(x, w, R, N, pado, f"{cid} dense again", bias=bias, ln=ln)), f"{cid}: not deterministic"

    # the activations on the same pre-activation
    vd = v.double()
    gelu = run_gemv(x, w, R, N, pado, f"{cid} gelu_tanh", bias=bias, ln=ln, act=ops.ACT_GELU_TANH).double()
    gref = 0.5 * vd * (1 + torch.tanh(math.sqrt(2 / math.pi) * (vd + 0.044715 * torch.pow(vd, 3))))
    r_gelu = (gelu - gref).abs() / (2.0 ** -20 * vd.abs()).clamp_min(1e-300)
    assert worst(r_gelu) <= 1.0, f"{cid}: gelu_tanh err/bound {worst(r_gelu):.3g}"
    th = run_gemv(x, w, R, N, pado, f"{cid} tanh", bias=bias, ln=ln, act=ops.ACT_TANH).double()
    tref = torch.tanh(vd)
    r_tanh = (th - tref).abs() / (2.0 ** -22 * tref.abs()).clamp_min(1e-300)
    assert worst(r_tanh) <= 1.0, f"{cid}: tanh err/bound {worst(r_tanh):.3g}"

    # the residual add
    o0 = torch.randn(R, N, generator=g, device=DEV) * 4
    acc = run_gemv(x, w, R, N, pado, f"{cid} accumulate", bias=bias, ln=ln, accumulate=True, fill=o0)
    assert torch.equal(acc, o0 + v), f"{cid}: accumulate != fp32 o0 + v"

    REACHED.add(plan)
    RAN.add(cid)
    print(f"[textdec-cov] gemv {cid} (ks {plan[0]}, {plan[1]} iterations): worst err/bound dense {worst(r_dense):.3g}, "
          f"gelu_tanh {worst(r_gelu):.3g}, tanh {worst(r_tanh):.3g}; staged LayerNorm elements rounded across a midpoint "
          f"{flips} of {R * K}")


def test_every_path_reached():
    """the cases together reached every K-split, and more than one grid-stride iteration at ks 1 and at ks 8"""
    if _num_sms() != SMS_LAYOUT:
        pytest.skip(f"tables laid out for {SMS_LAYOUT} SMs")
    if RAN != {c["id"] for c in GEMV_CASES}:
        pytest.skip("runs after the whole case table")
    assert {ks for ks, _ in REACHED} == {1, 2, 4, 8}, sorted(REACHED)
    for ks in (1, 8):
        assert any(k == ks and it > 1 for k, it in REACHED), f"no multi-iteration grid stride at ks {ks}: {sorted(REACHED)}"


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_textdec_attention
# ---------------------------------------------------------------------------------------------------------------------------
ATT_SCALE = 0.125
ATT_LAYERS, ATT_LAYER = 3, 1      # mem is this layer's column slice of [R, layers * H * 64]
ATT_CASES = [(16, 12, 32, s) for s in (0, 1, 13, 31)] + [(3, 5, 9, s) for s in (0, 1, 4, 8)]


def att_inputs(R, H, T, s, seed):
    """qkv [R, 3 D] in a NaN-padded [R, 3 D + 40] buffer (q ~ N(0, 12^2): scores of std ~12), mem the ATT_LAYER slice of a
    NaN-filled [R, ATT_LAYERS D], caches [R, H, T, 64] random below slot s and NaN from s on.  Pairs w = r H + h with w % 3 == 1
    get a latent key of score 45 along q, w % 3 == 2 a new key of score 45."""
    D = H * 64
    g = _gen(seed)
    q = torch.randn(R, H, 64, generator=g, device=DEV) * 12
    kn = torch.randn(R, H, 64, generator=g, device=DEV)
    vn = torch.randn(R, H, 64, generator=g, device=DEV)
    lat = torch.randn(R, H, 64, generator=g, device=DEV)
    top = q * (45.0 / (ATT_SCALE * q.square().sum(-1, keepdim=True)))
    w = (torch.arange(R * H, device=DEV) % 3).view(R, H, 1)
    lat = torch.where(w == 1, top, lat)
    kn = torch.where(w == 2, top, kn)
    qkv_buf = torch.full((R, 3 * D + 40), float("nan"), device=DEV)
    qkv_buf[:, :3 * D] = torch.cat([q.reshape(R, D), kn.reshape(R, D), vn.reshape(R, D)], 1)
    mem_buf = torch.full((R, ATT_LAYERS * D), float("nan"), device=DEV)
    mem_buf[:, ATT_LAYER * D:(ATT_LAYER + 1) * D] = lat.reshape(R, D)
    kc = torch.randn(R, H, T, 64, generator=g, device=DEV)
    vc = torch.randn(R, H, T, 64, generator=g, device=DEV)
    kc[:, :, s:] = float("nan")
    vc[:, :, s:] = float("nan")
    return q, kn, vn, lat, qkv_buf, mem_buf, kc, vc


def att_reference(q, kn, vn, lat, kc, vc, s):
    """fp64 output [R, H, 64] and the per-element bound of the module docstring"""
    qd = q.double()
    keys = torch.cat([lat[:, :, None], kc[:, :, :s], kn[:, :, None]], 2).double()      # [R, H, n, 64]
    vals = torch.cat([lat[:, :, None], vc[:, :, :s], vn[:, :, None]], 2).double()
    n = s + 2
    sc = (keys * qd[:, :, None]).sum(-1) * ATT_SCALE                                    # [R, H, n]
    p = sc.softmax(-1)
    ref = (p[..., None] * vals).sum(2)

    def xerr(a):
        return 2.0 ** -23 * (2 + 1.173 * a) + U * a

    E = 7 * U * ATT_SCALE * (keys.abs() * qd.abs()[:, :, None]).sum(-1)
    m = sc.cummax(-1).values
    step = xerr(m[..., 1:] - m[..., :-1]) * (m[..., 1:] > m[..., :-1])
    S = torch.zeros_like(sc)
    S[..., :-1] = step.flip(-1).cumsum(-1).flip(-1)
    d = E + xerr(m - sc) + S
    bound = ((p * d)[..., None] * (vals - ref[:, :, None]).abs()).sum(2)
    bound += 2 * n * U * (p[..., None] * vals.abs()).sum(2) + (n + 1) * U * ref.abs()
    return ref, bound, sc


@pytest.mark.parametrize("R,H,T,s", ATT_CASES)
def test_attention_step(R, H, T, s):
    ops = _ops()
    D = H * 64
    q, kn, vn, lat, qkv_buf, mem_buf, kc, vc = att_inputs(R, H, T, s, seed=R * 100 + H * 10 + s)
    kc0, vc0 = kc.clone(), vc.clone()
    out_buf = torch.full((R, D + 32), SENTINEL, device=DEV)
    step = torch.tensor([s], dtype=torch.int32, device=DEV)
    ops.textdec_attention(qkv_buf[:, :3 * D], mem_buf[:, ATT_LAYER * D:(ATT_LAYER + 1) * D], kc, vc, step, out_buf[:, :D],
                          scale=ATT_SCALE)
    what = f"attention R {R} H {H} T {T} s {s}"
    assert (out_buf[:, D:] == SENTINEL).all(), f"{what}: wrote past the out rows"
    out = out_buf[:, :D].reshape(R, H, 64)
    assert torch.isfinite(out).all(), f"{what}: non-finite output (a NaN slot was read)"

    # the cache: slot s holds this step's k / v, every other slot is unchanged bit for bit (NaNs included)
    assert torch.equal(kc[:, :, s], kn) and torch.equal(vc[:, :, s], vn), f"{what}: slot {s} does not hold this step's k / v"
    keep = torch.ones(T, dtype=torch.bool, device=DEV)
    keep[s] = False
    for c, c0, name in ((kc, kc0, "kcache"), (vc, vc0, "vcache")):
        assert torch.equal(c[:, :, keep].view(torch.int32), c0[:, :, keep].view(torch.int32)), f"{what}: {name} changed off slot {s}"

    ref, bound, sc = att_reference(q, kn, vn, lat, kc0, vc0, s)
    am = sc.argmax(-1)
    assert (am == 0).any() and (am == s + 1).any() and sc.abs().amax() > 35, f"{what}: the inputs miss a maximum position"
    ratio = (out.double() - ref).abs() / bound
    print(f"[textdec-cov] {what}: worst err/bound {worst(ratio):.3g}, scores in [{sc.min().item():.1f}, {sc.max().item():.1f}]")
    assert worst(ratio) <= 1.0, f"{what}: err/bound {worst(ratio):.3g} at {torch.unravel_index(ratio.argmax(), ratio.shape)}"


@pytest.mark.parametrize("s", [9, 10])
def test_attention_step_out_of_range(s):
    """*step >= T writes nothing: out and both caches stay as they were"""
    ops = _ops()
    R, H, T = 3, 5, 9
    D = H * 64
    _, _, _, _, qkv_buf, mem_buf, kc, vc = att_inputs(R, H, T, T - 1, seed=s)
    kc0, vc0 = kc.clone(), vc.clone()
    out = torch.full((R, D), SENTINEL, device=DEV)
    ops.textdec_attention(qkv_buf[:, :3 * D], mem_buf[:, ATT_LAYER * D:(ATT_LAYER + 1) * D], kc, vc,
                          torch.tensor([s], dtype=torch.int32, device=DEV), out, scale=ATT_SCALE)
    assert (out == SENTINEL).all()
    assert torch.equal(kc.view(torch.int32), kc0.view(torch.int32)) and torch.equal(vc.view(torch.int32), vc0.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_textdec_embed
# ---------------------------------------------------------------------------------------------------------------------------
EMBED_CASES = [  # (R, D, V, P, pos_offset, s)
    (16, 768, 300, 40, 1, 0), (16, 768, 300, 40, 1, 17), (1, 768, 300, 40, 0, 5),
    (16, 200, 50, 12, 1, 11), (1, 200, 50, 12, 0, 30),                     # s + pos_offset >= P: clamped to P - 1
]


@pytest.mark.parametrize("R,D,V,P,off,s", EMBED_CASES)
def test_embed(R, D, V, P, off, s):
    """(wte[tok] + wpe[s + pos_offset]) + emb in fp32, bitwise; tokens [R, 33] (the decoder's row stride), row 0 holds -1 and
    row R - 1 (when R > 2) V + 5 at column s"""
    ops = _ops()
    g = _gen(R * 1000 + D + s)
    wte = torch.randn(V, D, generator=g, device=DEV)
    wpe = torch.randn(P, D, generator=g, device=DEV) * 0.1
    emb = torch.randn(R, D, generator=g, device=DEV) * 3
    tokens = torch.randint(0, V, (R, 33), generator=g, device=DEV, dtype=torch.int32)
    tokens[0, s] = -1
    if R > 2:
        tokens[R - 1, s] = V + 5
    out = torch.full((R, D), SENTINEL, device=DEV)
    ops.textdec_embed(tokens, torch.tensor([s], dtype=torch.int32, device=DEV), wte, wpe, emb, out, pos_offset=off)
    tok = tokens[:, s].long().clamp(0, V - 1)
    ref = (wte[tok] + wpe[min(s + off, P - 1)][None, :]) + emb
    assert torch.equal(out, ref), f"embed R {R} D {D} s {s} pos_offset {off}: {int((out != ref).sum())} elements differ"


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_textdec_sample: bookkeeping
# ---------------------------------------------------------------------------------------------------------------------------
SV, SLDL, SEOS, SMAXLEN, SR = 40, 48, 17, 30, 5
DONE_ROW, EOS_ROW = 1, 2


@pytest.mark.parametrize("mode", ["uniforms", "forced"])
@pytest.mark.parametrize("s", [3, SMAXLEN - 3])
def test_sample_bookkeeping(s, mode):
    """5 rows over V = 40 logits in a [5, 48] buffer with NaN padding: row 1 is finished, row 2 draws (or is forced) <eos>, the
    others draw (or are forced) an ordinary token.  At s = max_len - 3 those get the closing <eos> at s + 2."""
    ops = _ops()
    g = _gen(s * 2 + (mode == "forced"))
    temperature = 0.7
    buf = torch.full((SR, SLDL), float("nan"), device=DEV)
    logits = buf[:, :SV]
    logits.copy_(torch.randn(SR, SV, generator=g, device=DEV))
    logits[EOS_ROW, SEOS] = 3.0
    tokens0 = (1000 + torch.arange(SR * 33, device=DEV, dtype=torch.int32)).view(SR, 33)
    lengths0 = 90 + torch.arange(SR, device=DEV, dtype=torch.int32)
    done0 = torch.zeros(SR, dtype=torch.int32, device=DEV)
    done0[DONE_ROW] = 1
    tokens, lengths, done = tokens0.clone(), lengths0.clone(), done0.clone()
    record = torch.full((32, SR, SV), SENTINEL, device=DEV)
    step = torch.tensor([s], dtype=torch.int32, device=DEV)

    # the token each row should get: an ordinary one (not <eos>) of probability > 1%, <eos> on EOS_ROW
    p = torch.softmax(logits.double() / temperature, -1)
    want = []
    for r in range(SR):
        if r == EOS_ROW:
            want.append(SEOS)
        else:
            cand = [t for t in (p[r] > 0.01).nonzero().flatten().tolist() if t != SEOS]
            want.append(cand[(3 * r + s) % len(cand)])
    if mode == "uniforms":
        cdf = torch.cat([torch.zeros(SR, 1, dtype=torch.float64, device=DEV), p.cumsum(-1)], 1)
        u = torch.rand(SR, 32, generator=g, device=DEV, dtype=torch.float64)
        for r, t in enumerate(want):
            u[r, s] = (cdf[r, t] + cdf[r, t + 1]) / 2 / cdf[r, -1]           # the middle of token t's interval
        ops.textdec_sample(logits, tokens, done, lengths, step, temperature=temperature, uniforms=u, eos=SEOS, max_len=SMAXLEN,
                           record=record)
    else:
        forced = torch.randint(0, SV, (SR, 35), generator=g, device=DEV, dtype=torch.int32)
        for r, t in enumerate(want):
            forced[r, s + 1] = t
        ops.textdec_sample(logits, tokens, done, lengths, step, temperature=temperature, forced=forced, eos=SEOS,
                           max_len=SMAXLEN, record=record)

    rec_want = torch.full_like(record, SENTINEL)
    rec_want[s] = logits
    assert torch.equal(record, rec_want), "record must hold this step's logits at [s][r][:V] and nothing else"
    tw, lw, dw = tokens0.clone(), lengths0.clone(), done0.clone()
    for r in range(SR):
        if r == DONE_ROW:
            continue
        tw[r, s + 1] = want[r]
        if want[r] == SEOS:
            dw[r], lw[r] = 1, s + 2
        elif s + 1 >= SMAXLEN - 2:
            tw[r, s + 2], dw[r], lw[r] = SEOS, 1, s + 3
    assert torch.equal(tokens, tw), (tokens[:, s:s + 3].tolist(), tw[:, s:s + 3].tolist())
    assert torch.equal(lengths, lw), (lengths.tolist(), lw.tolist())
    assert torch.equal(done, dw), (done.tolist(), dw.tolist())
