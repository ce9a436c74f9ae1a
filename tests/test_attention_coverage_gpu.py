"""The flash attention (attention.cu) element by element against fp64, at every kernel instantiation, its masks, the ring
stages and wraps of its key pipeline, the lazy softmax rescale, and every launch of the UNet step.

Dispatch.  The C ABI picks an instantiation from d_head (a multiple of 8) through vdb_attention_dk_pad / dv_pad; INSTANCES
restates it and each case asserts that the pads agree:
    d_head    DK   DVP  BKV  stages  form
    8-48      64   48   128  3       consumer-issued TMA
    56-64     64   64   128  2       consumer-issued TMA
    72-80     128  80   64   3       consumer-issued TMA
    136-160   192  160  64   2       producer warp
    64        64   64   128  2       varlen (vdb_attention_varlen_bf16)
d_head 88-128 and > 160 are refused (test_cabi pins that).  Key tile t sits in ring stage t % stages and waits for phase
(t / stages) & 1, so a batch item with n keys runs T = ceil(n / BKV) tiles and wraps its rings (T - 1) // stages times.  Each
case is tagged with the instantiation, T, the wraps, the keys in its last tile, whether the last 128-row query tile is partial
and whether that tile of item b reads rows of item b + 1 (B >= 2 and ceil(Nq / 128) 128 > q_bstride).

Notation: u = 2^-24; c = float32(scale) log2(e) in exact arithmetic; c^ = fl(scale * 1.4426950f), the kernel's scale_log2,
with |c^ - c| <= 2^-23 c (the rounded constant and the product, u each); Q = min(DVP, DK) / 16, the kernel's K16 steps of QK^T;
S_j the exact score of key j over the bf16 operands, M = max_j S_j and M_abs = max_j |S_j| over the row's visible keys; n the
visible keys and T the key tiles of the row's item.  Per-element bounds are first order: every neglected term is a product of
two of the relative errors below (each < 2^-8), so it is below 2^-8 of a first-order term that the bound already contains.

The kernel, per row: s_j = S_j with fp32 wgmma accumulation; per tile the running maximum m (a kernel score) is replaced only
when the tile maximum exceeds it by more than 8 log2 units, rescaling l and O by f = ex2((m_old - m_new) c^); otherwise m stays.
Each weight is P_j = ex2.approx.ftz(fmaf(s_j, c^, -fl(m c^))); l sums the fp32 P_j, O accumulates bf16(P_j) V_j in fp32
(wgmma), and out = bf16(O * (1 / l)).

Error sources (relative errors of the weight W_j = P_j times the later factors f, in log2 units first):
  (a) QK^T: bf16 x bf16 products are exact in fp32, and each of the Q mma steps rounds the running sum by at most 2^-22 of its
      magnitude: |s_j - S_j| <= Q 2^-22 A_j, A_j = sum_c |q_c k_jc|; times c^: c Q 2^-22 A_j.
  (b) c^ != c: (c^ - c) S_j, of which (c^ - c) M is common to all keys: 2^-23 c (M - S_j).
  (c) fl(m c^) errs by u |m c^| <= u c M_abs in each epoch of m (it does not cancel between epochs).
  (d) fmaf rounds its result x_j once, |x_j| <= c (M - S_j): u c (M - S_j).
  (e) the rescale arguments (one subtraction and one product, 2u each) sum over the epochs after key j's to at most
      2u c (M - S_j) (the maxima telescope from m >= S_j to M).
  (f) ex2.approx.ftz.f32: EPS_EX2 = 2^-22 relative, the documented 2 ulp maximum error of exp2f (the CUDA math API's
      exp2f is this instruction) over the full range, on P_j and on each of the at most T - 1 rescale factors applied to it:
      T EPS_EX2.  ex2 results below 2^-126 flush to zero: at most 2^-126 absolute per key, against l >= 1 (the key that set m
      has weight ~1, a later rescale gives the new maximum weight ~1).
  d_j = ln 2 [c Q 2^-22 A_j + (2^-23 + 3u) c (M - S_j) + u c M_abs] + T EPS_EX2   (relative, since 2^x - 1 <= x ln 2 (1 + x))
The same W_j feeds l and, rounded to bf16, O, so d_j is common to numerator and denominator and cancels up to
|sum_j p_j d_j (v_j - ref)| <= sum_j p_j d_j (|v_j| + |ref|) (p_j the fp64 softmax weights, ref = sum_j p_j v_j).  Then:
  (g) bf16(P_j) in the numerator only: EPS_P sum_j p_j |v_j|, EPS_P = 2^-8, the relative rounding error of round-to-nearest
      bf16 (8 significant bits).
  (h) O: T BKV / 16 wgmma steps of 2^-22 of the running magnitude <= sum_j W_j |v_j|, and up to T rescaling products, u each:
      (T BKV / 16 2^-22 + T u) sum_j p_j |v_j|.
  (i) l: each thread adds its BKV / 4 weights of a tile in BKV / 4 roundings, the rescales multiply it T times, two
      shuffle adds join the four threads of a row; all terms are positive: D_l u |ref|, D_l = T (BKV / 4 + 1) + 2.
  (j) 1 / l (IEEE division, the library is built without fast math) and the product by it: 2u |ref|.
  (k) the flushed weights: n 2^-126 (max_j |v_j| + |ref|).
So the fp32 value the epilogue rounds lies within
    e = sum_j p_j d_j (|v_j| + |ref|) + (EPS_P + T BKV / 16 2^-22 + T u) sum_j p_j |v_j| + (D_l + 2) u |ref| + n 2^-126 (..)
of ref, and round-to-nearest bf16 is monotone, so out must lie in [bf16(ref - e), bf16(ref + e)]: bf16(ref) itself except
where ref is within e of a rounding midpoint.  The printed err/bound is |out - ref| / (e + half a bf16 ulp of |ref| + e), which
the output rounding alone takes near 1; (|out - ref| - half a bf16 ulp of out) / e, also printed, is a lower bound on the
share of e the fp32 value used.

Exact power-of-two suite.  scale = float32(ln 2) makes c^ = fl(0.6931472f * 1.4426950f) = 1.0 exactly.  Each Q row is one-hot
(weight +-1) in a channel below d_head, K and V hold small integers (exact in bf16), so every s_j is an integer computed
exactly, fmaf and m c^ are exact, every P_j and every rescale factor is 2^integer up to ex2's error, and the reference is the
base-2 softmax of the integer scores, sum_j 2^(S_j - M) v_j / sum_j 2^(S_j - M), in fp64 (its own error, ~n 2^-53 relative,
is far below e).  (a)-(e) vanish: d_j = T EPS_EX2.  (g) shrinks to EPS_EX2: bf16(P_j) is the bf16 value nearest P_j, and
2^x_j is a bf16 value within EPS_EX2 P_j of it.  (h)-(k) stay.  Whether each output came out exactly bf16(ref) is printed,
not asserted.  Channels carry per-tile patterns (row r takes its pattern from PAIRS, so rows r and r + 8 of a 16-row fragment
group, held by one thread, differ): a ramp of +9 per tile (a rescale every tile), +7 per tile (every second tile), a single
jump of exactly +8 (no rescale: the test is strict; P reaches 2^8), a last key 200 above the rest (without the rescale P
overflows), the maximum at key 0 with the others 20-159 below (those under -126 flush), all scores equal (the exact mean of
V), and random small integers.  The reach table restates the rescale rule (a jump of more than 8 over the running maximum,
per BKV tile) only to count what the cases reached; the numeric checks hold for any correct kernel.

Random suite.  randn-like bf16 q, k, v with q scaled per head so that c S has a std of 0.7 to 17 log2 units (spreads up to
about +-60), against softmax(float32(scale) q k^T) v in fp64 with the bound e above.  The cases include every launch of the
UNet step (B 8, H 8: self-attention through the fused q | k buffer at N 4096 / 1024 / 256 / 64 with d_head 40 / 80 / 160 / 160,
cross-attention over 77 and 257 context tokens stored in 80 / 264 rows per item at each level), the ragged self-attention path
(kv_bstride = Np > N), CLIP's text (77 of 80 rows, causal, d 64, H 12) and image (257 of 264, d 64, H 16) encoders, a small
case at every supported d_head, causal masks at d_head 40, 80 and 160, and the varlen entry with kv_len 0, 1, 127, 128,
129, 248, Nk, > Nk (clamped) and negative (an item without visible keys must get zero rows).

Layout and write safety, every case: Q and K sit in wider buffers (NaN in the columns outside the heads; ldq != ldk; in the
fused q | k buffer the columns after the K half), V^T has NaN columns past B kv_bstride, out is a row-strided view with
sentinel columns on both sides (the right band wider than DVP - d_head), sentinel rows in [Nq, q_bstride) of every item and
a margin of more than one query tile after the last item: all sentinels must survive bitwise.  Pad keys [n, kv_bstride) and
pad query rows [Nq, q_bstride) hold +-3e38; the output must be bitwise that of a run with zero padding, and a second launch
must reproduce it bitwise.  The pads the header requires to be zero (Q / K channels past d_head, V^T rows past d_head) stay
zero.
"""
import math
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
U = 2.0 ** -24
EPS_EX2 = 2.0 ** -22          # (f); a polynomial exp2 on the FMA pipe would put its own relative error here
EPS_P = 2.0 ** -8             # (g)
FTZ = 2.0 ** -126             # (k)
LOG2E = 1.0 / math.log(2.0)
SCALE_EXACT = float(np.float32(math.log(2.0)))   # c^ = 1.0 exactly
GARBAGE = 3.0e38
SENTINEL = -7777.0
KBQ = 128

# name: (DK, DVP, BKV, stages)
INSTANCES = {"dvp48": (64, 48, 128, 3), "dvp64": (64, 64, 128, 2), "dvp80": (128, 80, 64, 3), "dvp160": (192, 160, 64, 2),
             "varlen": (64, 64, 128, 2)}
DISPATCH_TAGS = ("1 tile", "fewer tiles than stages", "2 ring wraps", "tail 8", "tail BKV-8", "partial query tile",
                 "cross-item Q read")
RESCALE_TAGS = ("0 rescales", "1 rescale", ">=2 rescales", "jump of exactly 8", "jump of 200", "row0 rescales, row0+8 not",
                "row0+8 rescales, row0 not")
REACHED = {k: set() for k in INSTANCES}
RESCALED = {k: set() for k in INSTANCES}
RAN = set()
WORST = {}                    # (suite, instantiation) -> worst err/bound


def _ops():
    from vdb200 import ops
    return ops


def instance_of(d, varlen=False):
    if varlen:
        return "varlen"
    if 8 <= d <= 48:
        return "dvp48"
    if d <= 64:
        return "dvp64"
    if d <= 80:
        return "dvp80"
    if 136 <= d <= 160:
        return "dvp160"
    raise ValueError(d)


def _case(cid, B, H, Nq, Nk, d, qbs=0, kvbs=0, causal=False, fused=False, suites=("rand",), kv_len=None, cols=(64, 128)):
    return dict(id=cid, B=B, H=H, Nq=Nq, Nk=Nk, d=d, qbs=qbs or Nq, kvbs=kvbs or Nk, causal=causal, fused=fused,
                suites=suites, kv_len=kv_len, cols=cols)


VARLEN_LENS = [0, 1, 127, 128, 129, 248, 520, 570, -3]
CASES = [
    # exact power-of-two suite: per instantiation a long case (>= 2 ring wraps, 8-key tail, partial query tile of 72 rows in
    # 80-row items), a short one (fewer tiles than stages, BKV - 8 key tail) and, where that differs, a one-tile case
    _case("x-d40-wrap", 2, 2, 72, 776, 40, qbs=80, kvbs=784, suites=("exact",)),
    _case("x-d40-two", 1, 2, 128, 248, 40, kvbs=256, suites=("exact",), cols=(32, 72)),
    _case("x-d8-one", 1, 2, 64, 8, 8, kvbs=16, suites=("exact",), cols=(16, 40)),
    _case("x-d64-wrap", 2, 2, 72, 520, 64, qbs=80, kvbs=528, suites=("exact",)),
    _case("x-d56-one", 1, 2, 128, 120, 56, kvbs=128, suites=("exact",), cols=(32, 72)),
    _case("x-d80-wrap", 2, 2, 72, 392, 80, qbs=80, kvbs=400, suites=("exact",)),
    _case("x-d72-two", 1, 2, 128, 120, 72, kvbs=128, suites=("exact",), cols=(32, 72)),
    _case("x-d80-one", 1, 1, 40, 8, 80, kvbs=16, suites=("exact",)),
    _case("x-d160-wrap", 2, 2, 72, 264, 160, qbs=80, kvbs=272, suites=("exact",)),
    _case("x-d144-one", 1, 2, 128, 56, 144, kvbs=64, suites=("exact",), cols=(32, 72)),
    # varlen: both suites, Nq != Nk, every kv_len edge
    _case("varlen", len(VARLEN_LENS), 2, 200, 520, 64, qbs=208, kvbs=528, suites=("exact", "rand"), kv_len=VARLEN_LENS),
    # the UNet step (B 8, H 8): fused self-attention and both context lengths at every level
    _case("unet-self-4096-d40", 8, 8, 4096, 4096, 40, fused=True),
    _case("unet-self-1024-d80", 8, 8, 1024, 1024, 80, fused=True),
    _case("unet-self-256-d160", 8, 8, 256, 256, 160, fused=True),
    _case("unet-self-64-d160", 8, 8, 64, 64, 160, fused=True),
] + [
    _case(f"unet-cross-{N}-d{d}-L{L}", 8, 8, N, L, d, kvbs=(L + 7) // 8 * 8)
    for N, d in ((4096, 40), (1024, 80), (256, 160), (64, 160)) for L in (77, 257)
] + [
    _case("ragged-self-625-d40", 2, 8, 625, 625, 40, kvbs=632),
    _case("clip-text", 2, 12, 77, 77, 64, qbs=80, kvbs=80, causal=True, fused=True),
    _case("clip-image", 2, 16, 257, 257, 64, qbs=264, kvbs=264, fused=True),
    _case("causal-d40-fused", 2, 2, 333, 333, 40, qbs=336, kvbs=336, causal=True, fused=True),
    _case("causal-d80", 2, 3, 300, 300, 80, kvbs=304, causal=True),
    _case("causal-d160", 1, 2, 200, 200, 160, causal=True, cols=(32, 72)),
] + [
    _case(f"small-d{d}", 2, 2, 100, 300, d, qbs=104, kvbs=304, cols=(32, 72))
    for d in (8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 136, 144, 152, 160)
]


def visible(case):
    """keys visible to each item"""
    if case["kv_len"] is None:
        return [case["Nk"]] * case["B"]
    return [max(0, min(n, case["Nk"])) for n in case["kv_len"]]


def dispatch_tags(case, inst):
    _, _, BKV, stages = INSTANCES[inst]
    tags = set()
    for n in visible(case):
        if n == 0:
            continue
        T = -(-n // BKV)
        tail = n - (T - 1) * BKV
        if T == 1:
            tags.add("1 tile")
        if T < stages:
            tags.add("fewer tiles than stages")
        if (T - 1) // stages >= 2:
            tags.add("2 ring wraps")
        if tail == 8:
            tags.add("tail 8")
        if tail == BKV - 8:
            tags.add("tail BKV-8")
    if case["Nq"] % KBQ:
        tags.add("partial query tile")
    if case["B"] >= 2 and -(-case["Nq"] // KBQ) * KBQ > case["qbs"]:
        tags.add("cross-item Q read")
    return tags


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


ALPHAS = (0.5, 2.0, 6.0, 12.0)     # q std per head (cycled): c S has a std of 1.44 alpha log2 units


def random_inputs(case, seed):
    """fp32 (bf16-exact) q [B, H, Nq, d], k / v [B, H, Nk, d]"""
    B, H, Nq, Nk, d = case["B"], case["H"], case["Nq"], case["Nk"], case["d"]
    g = _gen(seed)
    alpha = torch.tensor([ALPHAS[h % len(ALPHAS)] for h in range(H)], device=DEV).view(1, H, 1, 1)
    q = (torch.randn(B, H, Nq, d, generator=g, device=DEV) * alpha).to(BF16).float()
    k = torch.randn(B, H, Nk, d, generator=g, device=DEV).to(BF16).float()
    v = torch.randn(B, H, Nk, d, generator=g, device=DEV).to(BF16).float()
    return q, k, v


# channel patterns of the exact suite (channel c < 8 of K); row r of a 16-row fragment group reads PAIRS[...][r // 8 % 2]
RAMP9, RAMP7, JUMP8, LATE200, MAX0, CONST, RAND4, RAND30 = range(8)
PAIRS = [(RAMP9, CONST), (CONST, RAMP9), (RAMP7, JUMP8), (JUMP8, RAMP7), (LATE200, MAX0), (MAX0, LATE200), (RAND30, RAND4),
         (RAMP9, JUMP8)]


def exact_inputs(case, inst, seed):
    """q one-hot (weight -1 on every fourth 16-row group, else +1) on the pattern channel of its row; k per pattern over the
    item's visible keys (LATE200 puts 200 on the last visible key); v small integers"""
    B, H, Nq, Nk, d = case["B"], case["H"], case["Nq"], case["Nk"], case["d"]
    BKV = INSTANCES[inst][2]
    g = _gen(seed)
    j = torch.arange(Nk, device=DEV)
    t, i = j // BKV, j % BKV
    k = torch.randint(-4, 5, (B, H, Nk, d), generator=g, device=DEV).float()
    for b, n in enumerate(visible(case)):
        kb = k[b]
        kb[:, :, RAMP9] = (9 * t - i % 4).float()
        kb[:, :, RAMP7] = (7 * t - i % 3).float()
        kb[:, :, JUMP8] = -(i % 2).float()
        if Nk > BKV + 5:
            kb[:, BKV + 5, JUMP8] = 8.0
        kb[:, :, LATE200] = -(i % 3).float()
        if n > 0:
            kb[:, n - 1, LATE200] = 200.0
        kb[:, :, MAX0] = (-20 - j % 140).float()
        kb[:, 0, MAX0] = 0.0
        kb[:, :, CONST] = 0.0
        kb[:, :, RAND30] = torch.randint(-30, 31, (H, Nk), generator=g, device=DEV).float()
    assert torch.equal(k, k.to(BF16).float())
    r = torch.arange(Nq, device=DEV)
    q = torch.zeros(B, H, Nq, d, device=DEV)
    for b in range(B):
        for h in range(H):
            shift = (b * H + h) % len(PAIRS)
            ch = torch.tensor([PAIRS[(x % 8 + shift) % 8][x // 8 % 2] for x in range(16)], device=DEV)[r % 16]
            w = torch.where((r // 16) % 4 == 3, -1.0, 1.0)
            q[b, h, r, ch] = w
    v = torch.randint(-8, 9, (B, H, Nk, d), generator=g, device=DEV).float()
    return q, k, v


def layout(case, inst, q, k, v, pad):
    """the kernel's operands for q / k / v: (Q, K, Vt, q_col0, k_col0); pad keys and pad query rows hold `pad` (0 or
    random +-GARBAGE), every column outside the slices NaN, the header's zero pads zero"""
    B, H, Nq, Nk, d, qbs, kvbs = (case[x] for x in ("B", "H", "Nq", "Nk", "d", "qbs", "kvbs"))
    DK, DVP, _, _ = INSTANCES[inst]
    g = _gen(7)

    def fill(x):
        if pad == 0:
            return torch.zeros_like(x)
        return torch.where(torch.rand(x.shape, generator=g, device=DEV) < 0.5, -GARBAGE, GARBAGE).to(x.dtype)

    if case["fused"]:
        assert Nq == Nk and qbs == kvbs and case["kv_len"] is None
        buf = torch.full((B * qbs, 2 * H * DK + 16), float("nan"), dtype=BF16, device=DEV)
        qk = buf[:, :2 * H * DK].view(B, qbs, 2, H, DK)
        qk.zero_()
        qk[:, :Nq, 0, :, :d] = q.permute(0, 2, 1, 3).to(BF16)
        qk[:, :Nk, 1, :, :d] = k.permute(0, 2, 1, 3).to(BF16)
        qk[:, Nq:] = fill(qk[:, Nq:])
        Q, K, qc, kc = buf, buf, 0, H * DK
    else:
        qc, kc = case["cols"]
        Q = torch.full((B * qbs, qc + H * DK + 24), float("nan"), dtype=BF16, device=DEV)
        K = torch.full((B * kvbs, kc + H * DK + 40), float("nan"), dtype=BF16, device=DEV)
        qv = Q[:, qc:qc + H * DK].view(B, qbs, H, DK)
        kv = K[:, kc:kc + H * DK].view(B, kvbs, H, DK)
        qv.zero_()
        kv.zero_()
        qv[:, :Nq, :, :d] = q.permute(0, 2, 1, 3).to(BF16)
        kv[:, :Nk, :, :d] = k.permute(0, 2, 1, 3).to(BF16)
        qv[:, Nq:] = fill(qv[:, Nq:])
        for b, n in enumerate(visible(case)):
            kv[b, n:] = fill(kv[b, n:])
    Vt = torch.full((H * DVP, B * kvbs + 24), float("nan"), dtype=BF16, device=DEV)
    vv = Vt[:, :B * kvbs].view(H, DVP, B, kvbs)
    vv.zero_()
    vv[:, :d, :, :Nk] = v.permute(1, 3, 0, 2).to(BF16)
    for b, n in enumerate(visible(case)):
        vv[:, :d, b, n:] = fill(vv[:, :d, b, n:])
    return Q, K, Vt, qc, kc


def out_frame(case, inst):
    """(sentinel buffer, the out view, mask of the elements the kernel must write)"""
    B, H, Nq, d, qbs = (case[x] for x in ("B", "H", "Nq", "d", "qbs"))
    DVP = INSTANCES[inst][1]
    left, top = 8, 2
    right = (DVP - d + 15) // 8 * 8
    rows = top + B * qbs + KBQ + 2
    buf = torch.full((rows, left + H * d + right), SENTINEL, dtype=BF16, device=DEV)
    out = buf[top:top + B * qbs, left:left + H * d]
    mask = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    for b in range(B):
        mask[top + b * qbs:top + b * qbs + Nq, left:left + H * d] = True
    return buf, out, mask


def launch(case, inst, scale, ops_args):
    """one launch into a fresh sentinel frame; returns the output as [B, H, Nq, d] fp32 after checking the sentinels"""
    ops = _ops()
    Q, K, Vt, qc, kc, kv_len = ops_args
    B, H, Nq, Nk, d = (case[x] for x in ("B", "H", "Nq", "Nk", "d"))
    buf, out, mask = out_frame(case, inst)
    ops.attention(Q, K, Vt, out, B, H, Nq, Nk, d, scale=scale, q_col0=qc, k_col0=kc, causal=case["causal"],
                  q_bstride=case["qbs"], kv_bstride=case["kvbs"], kv_len=kv_len)
    torch.cuda.synchronize()
    sent = torch.tensor(SENTINEL, dtype=BF16).view(torch.int16).item()
    bad = (buf.view(torch.int16) != sent) & ~mask
    assert not bad.any(), f"{case['id']}: wrote outside the output slice, first at {tuple(bad.nonzero()[0].tolist())}"
    o = out.view(B, case["qbs"], H, d)[:, :Nq].permute(0, 2, 1, 3)
    return o.float().contiguous(), buf.clone()


# ---------------------------------------------------------------------------------------------------------------------------
# the fp64 reference and its bound, one (item, head) at a time
# ---------------------------------------------------------------------------------------------------------------------------
def reference(case, inst, q, k, v, b, h, exact, scale):
    """fp64 (ref [Nq, d], e [Nq, d], scores [Nq, n]) for item b, head h; None when the item has no visible key"""
    DK, DVP, BKV, _ = INSTANCES[inst]
    n = visible(case)[b]
    if n == 0:
        return None
    T = -(-n // BKV)
    Qs = min(DVP, DK) // 16
    qd, kd, vd = q[b, h].double(), k[b, h, :n].double(), v[b, h, :n].double()
    S = qd @ kd.t()
    Nq = S.shape[0]
    vis = torch.ones_like(S, dtype=torch.bool)
    if case["causal"]:
        vis = torch.arange(n, device=DEV)[None, :] <= torch.arange(Nq, device=DEV)[:, None]
    Sm = S.masked_fill(~vis, -math.inf)
    M = Sm.amax(1, keepdim=True)
    if exact:
        p = torch.exp2(Sm - M)
        dj = torch.full_like(S, T * EPS_EX2)
        num_round = EPS_EX2
    else:
        c = float(np.float32(scale)) * LOG2E
        p = torch.exp2(c * (Sm - M))
        A = qd.abs() @ kd.abs().t()
        M_abs = S.abs().masked_fill(~vis, 0).amax(1, keepdim=True)
        gap = (M - S).masked_fill(~vis, 0)
        dj = math.log(2) * (c * Qs * 2.0 ** -22 * A + (2.0 ** -23 + 3 * U) * c * gap + U * c * M_abs) + T * EPS_EX2
        num_round = EPS_P
    p = p / p.sum(1, keepdim=True)
    pd = (p * dj).masked_fill(~vis, 0)
    ref = p @ vd
    pv = p @ vd.abs()
    D_l = T * (BKV // 4 + 1) + 2
    e = (pd @ vd.abs() + ref.abs() * pd.sum(1, keepdim=True) + (num_round + T * BKV / 16 * 2.0 ** -22 + T * U) * pv
         + (D_l + 2) * U * ref.abs() + n * FTZ * (vd.abs().max() + ref.abs()))
    return ref, e, Sm


def half_ulp_bf16(x):
    _, ex = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), ex - 9)


def rescale_tags(Sm, BKV):
    """the kernel's lazy-rescale rule restated over the exact integer scores [Nq, n] of one (item, head)"""
    Nq, n = Sm.shape
    T = -(-n // BKV)
    pad = torch.full((Nq, T * BKV - n), -math.inf, dtype=Sm.dtype, device=DEV)
    tmax = torch.cat([Sm, pad], 1).view(Nq, T, BKV).amax(2)
    m = tmax[:, 0].clone()
    count = torch.zeros(Nq, dtype=torch.int64, device=DEV)
    tags = set()
    for t in range(1, T):
        jump = torch.clamp(tmax[:, t] - m, min=0)
        if (jump == 8).any():
            tags.add("jump of exactly 8")
        resc = jump > 8
        if (resc & (jump >= 200)).any():
            tags.add("jump of 200")
        count += resc
        m = torch.where(resc, tmax[:, t], m)
    for c, tag in ((0, "0 rescales"), (1, "1 rescale")):
        if (count == c).any():
            tags.add(tag)
    if (count >= 2).any():
        tags.add(">=2 rescales")
    r = torch.arange(Nq, device=DEV)
    lo = r[(r % 16 < 8) & (r + 8 < Nq)]
    if ((count[lo] > 0) & (count[lo + 8] == 0)).any():
        tags.add("row0 rescales, row0+8 not")
    if ((count[lo] == 0) & (count[lo + 8] > 0)).any():
        tags.add("row0+8 rescales, row0 not")
    return tags


def check_suite(case, inst, suite, seed):
    exact = suite == "exact"
    B, H, d = case["B"], case["H"], case["d"]
    DK, DVP, BKV, _ = INSTANCES[inst]
    scale = SCALE_EXACT if exact else d ** -0.5
    q, k, v = exact_inputs(case, inst, seed) if exact else random_inputs(case, seed)
    kv_len = None
    if case["kv_len"] is not None:
        kv_len = torch.tensor(case["kv_len"], dtype=torch.int32, device=DEV)
    args = (*layout(case, inst, q, k, v, GARBAGE), kv_len)
    out, frame = launch(case, inst, scale, args)
    out2, frame2 = launch(case, inst, scale, args)
    assert torch.equal(frame.view(torch.int16), frame2.view(torch.int16)), f"{case['id']} {suite}: not bitwise repeatable"
    del args
    _, frame0 = launch(case, inst, scale, (*layout(case, inst, q, k, v, 0), kv_len))
    assert torch.equal(frame.view(torch.int16), frame0.view(torch.int16)), \
        f"{case['id']} {suite}: the +-3e38 pad keys / pad query rows changed the output (against zero padding)"

    worst, used, not_rn, tags = 0.0, 0.0, 0, set()
    for b in range(B):
        for h in range(H):
            o = out[b, h].double()
            res = reference(case, inst, q, k, v, b, h, exact, scale)
            where = f"{case['id']} {suite} item {b} head {h}"
            if res is None:
                assert torch.equal(o, torch.zeros_like(o)), f"{where}: an item without visible keys must get zero rows"
                continue
            ref, e, Sm = res
            assert torch.isfinite(o).all(), f"{where}: non-finite output"
            lo, hi = (ref - e).to(BF16).double(), (ref + e).to(BF16).double()
            bad = (o < lo) | (o > hi)
            if bad.any():
                r, ch = divmod(int(bad.flatten().nonzero()[0]), d)
                raise AssertionError(f"{where}: {int(bad.sum())} outputs outside [bf16(ref - e), bf16(ref + e)]; first at row {r} "
                                     f"channel {ch}: got {o[r, ch].item():.8g}, fp64 {ref[r, ch].item():.8g}, e {e[r, ch].item():.3g}")
            ratio = (o - ref).abs() / (e + half_ulp_bf16(ref.abs() + e))
            worst = max(worst, ratio.max().item())
            used = max(used, (((o - ref).abs() - half_ulp_bf16(o)).clamp_min(0) / e).max().item())
            not_rn += int((o != ref.to(BF16).double()).sum())
            if exact:
                tags |= rescale_tags(Sm, BKV)
    key = (suite, inst)
    WORST[key] = tuple(max(a, b) for a, b in zip(WORST.get(key, (0.0, 0.0)), (worst, used)))
    if exact:
        RESCALED[inst] |= tags
    print(f"[attn-cov] {case['id']} ({inst}) {suite}: worst err/bound {worst:.3g}, fp32 error beyond the output rounding "
          f">= {used:.3g} e; outputs != bf16(fp64) {not_rn} of "
          f"{out.numel()}" + (f"; rescale paths {sorted(tags)}" if exact else ""))


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_attention_case(case):
    ops = _ops()
    inst = instance_of(case["d"], case["kv_len"] is not None)
    DK, DVP, _, _ = INSTANCES[inst]
    assert ops.attention_pads(case["d"]) == (DK, DVP), f"{case['id']}: the restated dispatch disagrees with the pads"
    for s, suite in enumerate(case["suites"]):
        check_suite(case, inst, suite, seed=zlib.crc32(case["id"].encode()) % 10000 + s)
    REACHED[inst] |= dispatch_tags(case, inst)
    RAN.add(case["id"])


def test_every_path_reached():
    """every instantiation saw one tile, fewer tiles than stages, two ring wraps, 8- and (BKV - 8)-key tails, a partial query
    tile and a cross-item Q read; and, in the exact suite, rows with 0, 1 and >= 2 rescales, a jump of exactly 8, a jump of
    200 and fragment-row pairs that rescale apart"""
    if RAN != {c["id"] for c in CASES}:
        pytest.skip("runs after the whole case table")
    for name in sorted(WORST):
        print(f"[attn-cov] {name[0]} {name[1]}: worst err/bound {WORST[name][0]:.3g}, fp32 error beyond the output rounding "
              f">= {WORST[name][1]:.3g} e")
    for inst in INSTANCES:
        missing = set(DISPATCH_TAGS) - REACHED[inst]
        assert not missing, f"{inst}: never reached {sorted(missing)}"
        missing = set(RESCALE_TAGS) - RESCALED[inst]
        assert not missing, f"{inst}: the exact suite never reached {sorted(missing)}"
