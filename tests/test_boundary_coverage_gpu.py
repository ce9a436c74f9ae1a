"""The kernels at the edges of every image call (elementwise.cu) element by element against fp64, or bit for bit against the
reference's own fp32 op: the CLIP text and image ends, the device CLIP preprocessing, the VAE's input and output ends, the
timestep embedding and the skinny time-MLP linear, the VAE mid-block softmax, the layout and cast kernels, and the PLMS and
img2img combinations.

Every capped elementwise grid is at most 16 CTAs of 256 threads per SM (ew_blocks); one item more than 16 * SMs * 256 runs the
grid-stride loop, so those sizes come from vdb_num_sms().  u = 2^-24 is fp32's unit roundoff; every bound below is first order and
multiplied by 1 + 2^-10 for the second-order terms.  Each case prints its max |err| and max |err| / bound.

Bitwise claims (no rounding differs from the reference's op):
  casts           __float2bfloat16 rounds to nearest even like torch's .to(bfloat16) (restated here on the CPU by c10's
                  bit trick), so ties (low half 0x8000) go to the even mantissa, the largest finite float rounds to inf, and
                  subnormals keep their bits; bf16 -> fp32 is exact.  NaN stays NaN (payloads may differ).
  upsample, patchify, mask_to_latent, clip_text_embed
                  copies, or one fp32 add then the same RNE to bf16; max_pool2d's rule (first maximum in row-major order, NaN
                  wins) is the kernel's.
  vit_assemble    (v + pos) * s in fp32, then RNE: the same two roundings as the reference's expression.
  im2col3x3_small bf16(x * s + t): with (s, t) = (1, 0) or (2, -1) the product is exact in fp32, so whether nvcc fuses it into an
                  FMA cannot change the result; pad taps and pad columns are exactly 0.
  permute         the decode's clamp((x + 1) / 2, 0, 1) as x * 0.5 + 0.5: division by 2 is exact outside subnormals, so
                  RN(x + 1) / 2 = RN((x + 1) / 2) = RN(0.5 x + 0.5), fused or not (0.5 x is exact), and x + 1 is either 0 or at
                  least 2^-24 in magnitude, never subnormal.
  axpby           __fadd_rn(__fmul_rn(a, x), __fmul_rn(b, z)): two products and one sum, the fp32 restatement a*x + b*z.
  clip_to_u8_hwc  truncation of RN(clamp(x, 0, 1) * 255), as (clamp(0, 1) * 255).byte(); inputs one fp32 ulp either side of
                  every k / 255 separate truncation from rounding.
  resample        integer arithmetic: each pass must equal oracle/pil_resample.py (pinned to Pillow on the CPU) on the same u8
                  input, and the chain its clip_preprocess.

Per-element bounds against fp64:
  timestep_embedding  the kernel computes e_k = RN(RN(-ln(max_period) * k) / half) in fp32 exactly as the reference does, so the
                  reference takes the same fp32 e_k (which keeps fp32's reading of ln 10^4 out of the bound) and evaluates
                  cos / sin(t exp(e_k)) in fp64.  expf is within 2 ulps (2^-22 relative) and t * f one rounding, so the argument
                  a errs by at most 1.25 * 2^-22 |a|; cosf / sinf add 2 ulps of a result <= 1:
                      |err| <= |a| 2^-21 + 2^-22.
                  An odd dim's last column is exactly 0, and the table + step_idx form equals the per-row form bit for bit.
  linear_small    each lane sums its ceil(K / 256) * 8 products in order, a 5-level shuffle tree folds the lanes, then the bias
                  is added: D = ceil(K / 256) * 8 + 6 roundings, |err| <= D u (sum_k |a_k w_k| + |b|) with a = act_in(x).
                  silu_f = __fdividef(x, 1 + __expf(-x)): __expf is within 2 + 1.173 |x| ulps and its argument's rounding adds
                  |x| u, 1 + e and __fdividef (2 ulps) the rest: (4 + |x|) 2^-23 relative.  With act_in that error enters as
                  sum_k |a_k w_k| (4 + |x_k|) 2^-23; with act_out the pre-activation error is multiplied by SiLU's slope
                  (< 1.1) and silu_f's own error is added at y.
  softmax_rows    per element and relative.  With A = max |x s| of the row, the argument z = x s - max errs by 3 A u, and
                  __expf(z) by (2 + 1.173 |z|) ulps <= (4 + 4.7 A) u: each exponential is within e = (4 + 8 A) u.  The sum of
                  positive terms (ceil(n / 256) in order per thread, a 5-level shuffle, 7 adds of the warp partials) adds
                  D = ceil(n / 256) + 12 u relative, the reciprocal and the product one u each:
                      eps = 2 e + (D + 2) u,   |y - p| <= 2^-8 (1 + eps) p + eps p
                  where 2^-8 p is the bf16 rounding of the output.  A row of equal logits at scale 1 has z = 0 exactly, so
                  every output is bf16(RN(1 / n)) bit for bit.
  scale_by_row_norm   the sum of squares of one row (ceil(C / 256) in order per thread, each maybe unfused: + 1, a 5-level
                  shuffle, 7 adds): D = ceil(C / 256) + 13 u relative; sqrtf halves it and adds u, the reciprocal, the product
                  and the row scale one u each:  |err| <= (D / 2 + 4) u |ref|.
  pointwise_small x * pre_mul rounds once, each product once (unless fused), and Cin sums:  |err| <= (Cin + 2) u (sum |w x pre| +
                  |b|).
  gaussian_sample from the fp32 moments: expf 2 ulps (4 u), the product, the sum and the post_mul product one u each:
                      |err| <= |post| (7 u |s n| + 2 u |m|),   s = exp(0.5 clamp(logvar, -30, 20)).
  lincomb4        y = c0 x0 (+ c1 x1 (+ c2 x2 (+ c3 x3))) in order, each product rounded or fused into the sum.  With t_i = c_i x_i
                  and S_k = t_0 + .. + t_k, the rounding of S_k errs by u |S_k| and an unfused product by u |t_i|:
                      |err| <= u (sum_k |S_k| + sum_{i >= 1} |t_i|).
                  This re-derives the flat 3 u sum |t_i|: at four terms the worst case of that sum order is 4 u |t_0| + 4 u |t_1|
                  + 3 u |t_2| + 2 u |t_3|, which 3 u sum |t_i| does not cover.  The coefficients reach the kernel as fp32; the
                  reference uses those fp32 values.

The coarser checks of test_kernels_gpu are kept as second guards.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
BF16 = torch.bfloat16
SLACK = 1.0 + 2.0 ** -10


def _ops():
    from vdb200 import ops
    return ops


def _sms():
    return int(_ops().lib.vdb_num_sms())


def ew_limit():
    """Items one pass of a capped elementwise grid covers (16 CTAs of 256 threads per SM); one more runs the grid-stride loop."""
    return 16 * _sms() * 256


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(*shape, generator=_gen(seed), device=DEV) * scale).to(dtype)


def _f32(v):
    return float(np.float32(v))


def check_bound(out, ref, bound, what):
    out, ref, bound = out.double(), ref.double(), bound.double() * SLACK
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs()
    bad = err > bound
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    print(f"{what}: max|err| {err.max().item():.3g}, max |err|/bound {ratio.max().item():.3g}")
    if bad.any():
        i = int((err - bound).argmax())
        idx = [int(j) for j in torch.unravel_index(torch.tensor(i), err.shape)]
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of bound; worst at {idx}: out "
                             f"{out.flatten()[i].item():.9g} ref {ref.flatten()[i].item():.9g} bound {bound.flatten()[i].item():.3g}")


_INT = {torch.float32: torch.int32, BF16: torch.int16, torch.uint8: torch.uint8}


def check_bitwise(out, ref, what):
    """Bit for bit, except that NaN payloads may differ (NaN must stay NaN)."""
    assert out.dtype == ref.dtype and out.shape == ref.shape, f"{what}: {out.dtype} {tuple(out.shape)} vs {ref.dtype} {tuple(ref.shape)}"
    out, ref = out.contiguous(), ref.to(out.device).contiguous()
    ob, rb = out.view(_INT[out.dtype]), ref.view(_INT[ref.dtype])
    if out.dtype.is_floating_point:
        on, rn = torch.isnan(out), torch.isnan(ref)
        assert torch.equal(on, rn), f"{what}: NaN at {int((on != rn).sum())} positions that disagree"
        diff = (ob != rb) & ~on
    else:
        diff = ob != rb
    print(f"{what}: {out.numel()} elements, {int(diff.sum())} differ in any bit")
    if diff.any():
        i = int(diff.flatten().nonzero()[0])
        idx = [int(j) for j in torch.unravel_index(torch.tensor(i), out.shape)]
        raise AssertionError(f"{what}: {int(diff.sum())} of {out.numel()} elements differ; first at {idx}: out "
                             f"{out.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_timestep_embedding
# ---------------------------------------------------------------------------------------------------------------------------
T_VALUES = (0, 1, 500, 981, 999)


@pytest.mark.parametrize("dim", [2, 64, 320, 321])
@pytest.mark.parametrize("B", [1, 8, 40])
def test_timestep_embedding(B, dim):
    ops = _ops()
    half = dim // 2
    nlp = torch.tensor(-math.log(10000), dtype=torch.float32)
    e = (torch.arange(half, dtype=torch.float32) * nlp) / torch.tensor(float(half), dtype=torch.float32)   # the reference's fp32 e_k
    freq = torch.exp(e.double()).to(DEV)
    for start in (range(len(T_VALUES)) if B < len(T_VALUES) else (0,)):
        ts = torch.tensor([T_VALUES[(start + i) % len(T_VALUES)] for i in range(B)], dtype=torch.int64, device=DEV)
        out = ops.timestep_embedding(ts, dim)
        a = ts.double()[:, None] * freq[None]
        ref = torch.cat([torch.cos(a), torch.sin(a)], -1)
        bound = torch.cat([a.abs(), a.abs()], -1) * 2.0 ** -21 + 2.0 ** -22
        if dim % 2:
            ref = torch.cat([ref, torch.zeros(B, 1, dtype=torch.float64, device=DEV)], -1)
            bound = torch.cat([bound, torch.zeros(B, 1, dtype=torch.float64, device=DEV)], -1)
            assert (out[:, -1].view(torch.int32) == 0).all(), "odd dim: last column is not +0"
        check_bound(out, ref, bound, f"timestep_embedding B{B} dim{dim} t0={T_VALUES[start]}")
    table = torch.tensor(T_VALUES, dtype=torch.int64, device=DEV)
    for j, t in enumerate(T_VALUES):
        idx = torch.tensor([j], dtype=torch.int32, device=DEV)
        per_row = ops.timestep_embedding(torch.full((B,), t, dtype=torch.int64, device=DEV), dim)
        check_bitwise(ops.timestep_embedding(table, dim, step_idx=idx, batch=B), per_row, f"timestep_embedding table t={t}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_linear_small
# ---------------------------------------------------------------------------------------------------------------------------
LS_MK = [(M, K) for M in (1, 2, 3, 8, 15, 16) for K in (8, 64, 320, 328, 1280)]


def _silu_err(v):
    return (4.0 + v.abs()) * 2.0 ** -23 * (v * torch.sigmoid(v)).abs()


@pytest.mark.parametrize("M,K", LS_MK)
def test_linear_small(M, K):
    ops = _ops()
    case = LS_MK.index((M, K))
    Ns = (1, 3, 5, 31, 33, 1280, 2 * _sms() * 32 + 37)          # the last runs the kernel's grid-stride loop over columns
    x = _randn(M, K, seed=case, scale=3.0)
    D = math.ceil(K / 256) * 8 + 6
    for j, N in enumerate(Ns):
        act_in, act_out = (j + case) & 1, ((j + case) >> 1) & 1
        with_bias = (j + case // 4) % 2 == 0
        w = _randn(N, K, seed=1000 + 10 * case + j, scale=K ** -0.5, dtype=BF16)
        b = _randn(N, seed=2000 + 10 * case + j) if with_bias else None
        out = ops.linear_small(x, w, b, act_in=act_in, act_out=act_out)
        xd, wd = x.double(), w.double()
        a = F.silu(xd) if act_in else xd
        bd = b.double() if with_bias else torch.zeros(N, dtype=torch.float64, device=DEV)
        y = a @ wd.t() + bd
        bound = D * U * (a.abs() @ wd.abs().t() + bd.abs())
        if act_in:
            bound = bound + ((4.0 + xd.abs()) * 2.0 ** -23 * a.abs()) @ wd.abs().t()
        ref = y
        if act_out:
            ref = F.silu(y)
            bound = 1.1 * bound + _silu_err(y)
        check_bound(out, ref, bound, f"linear_small M{M} K{K} N{N} act {act_in}/{act_out} bias {int(with_bias)}")


def test_linear_small_refuses_more_shared_memory_than_it_configures():
    from vdb200._lib import VdbError
    ops = _ops()
    x = torch.zeros(16, 3208, device=DEV)                          # 16 * 3208 * 4 B = 205,312 B > 200 KB
    w = torch.zeros(32, 3208, dtype=BF16, device=DEV)
    with pytest.raises(VdbError):
        ops.linear_small(x, w)


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_softmax_rows
# ---------------------------------------------------------------------------------------------------------------------------
VAE_SCALE = 512 ** -0.5
SM_CASES = [  # id, rows, n, scale, input std, sampled rows (None = all)
    ("vae-512sq", 4096, 4096, VAE_SCALE, 24.0, None),
    ("vae-panorama", 16384, 16384, VAE_SCALE, 24.0, 64),
    ("n1", 7, 1, 1.0, 2.0, None),
    ("n77", 5, 77, 1.0, 2.0, None),
    ("peaky-const", 300, 1000, 1.0, 2.0, None),
    ("row-stride", 2000, 257, 0.044, 40.0, None),                  # rows > 8 * SMs: the row grid-stride loop
]


def _softmax_bound(xs, p):
    """xs = x * s in fp64 [rows, n], p its fp64 softmax."""
    n = xs.shape[-1]
    A = xs.abs().amax(-1, keepdim=True)
    e = (4.0 + 8.0 * A) * U
    eps = 2 * e + (math.ceil(n / 256) + 12 + 2) * U
    return 2.0 ** -8 * (1 + eps) * p + eps * p


@pytest.mark.parametrize("cid,rows,n,scale,std,sampled", SM_CASES, ids=[c[0] for c in SM_CASES])
def test_softmax_rows(cid, rows, n, scale, std, sampled):
    ops = _ops()
    if cid == "row-stride":
        assert rows > 8 * _sms()
    x = _randn(rows, n, seed=rows + n, scale=std, dtype=BF16)
    if cid == "peaky-const":
        x[3] = _randn(n, seed=7, dtype=BF16)
        x[3, n // 3] = 40.0                                          # one logit +40 above a N(0, 1) row
        x[4] = 3.5                                                   # a constant row: every exponential exactly 1
    out = ops.softmax_rows(x, scale=scale)
    if sampled is None:
        sel = torch.arange(rows, device=DEV)
    else:
        sel = torch.randperm(rows - 2, generator=_gen(11), device=DEV)[:sampled - 2] + 1
        sel = torch.cat([torch.tensor([0, rows - 1], device=DEV), sel.sort().values])
    xs = x[sel].double() * _f32(scale)
    p = torch.softmax(xs, -1)
    check_bound(out[sel], p, _softmax_bound(xs, p), f"softmax_rows {cid} ({rows} x {n}, {sel.numel()} rows checked)")
    if cid == "peaky-const":
        inv = (torch.tensor(1.0, dtype=torch.float32) / n).to(BF16)
        check_bitwise(out[4], inv.expand(n).to(DEV), "softmax_rows constant row = bf16(RN(1/n))")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_clip_text_embed, vdb_patchify, vdb_vit_assemble, vdb_scale_by_row_norm
# ---------------------------------------------------------------------------------------------------------------------------
CLIP_VOCAB, CLIP_C = 49408, 768


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L,Lp", [(77, 80), (13, 16)])
def test_clip_text_embed(B, L, Lp):
    ops = _ops()
    tok = _randn(CLIP_VOCAB, CLIP_C, seed=1)
    pos = _randn(77, CLIP_C, seed=2, scale=0.1)
    ids = torch.randint(0, CLIP_VOCAB, (B, L), generator=_gen(3 + B), device=DEV)
    ids[:, :4] = torch.tensor([0, 49406, 49407, CLIP_VOCAB - 1], device=DEV)
    ids[-1, -1] = CLIP_VOCAB - 1
    out = ops.clip_text_embed(ids, tok, pos, Lp)
    ref = torch.zeros(B, Lp, CLIP_C, dtype=BF16, device=DEV)
    ref[:, :L] = (tok[ids] + pos[:L]).to(BF16)
    check_bitwise(out, ref, f"clip_text_embed B{B} L{L} Lp{Lp}")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("HW", [224, 28])
def test_patchify(B, HW):
    ops = _ops()
    P, kpad = 14, 640
    px = torch.rand(B, 3, HW, HW, generator=_gen(HW + B), device=DEV) * 4 - 2
    out = ops.patchify(px, P, kpad)
    cols = F.unfold(px, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)     # (c, py, px) columns, (gy, gx) rows
    ref = torch.zeros(cols.shape[0], kpad, dtype=BF16, device=DEV)
    ref[:, :3 * P * P] = cols.to(BF16)
    check_bitwise(out, ref, f"patchify B{B} {HW}^2")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("scale", ["none", "soft", "zeros"])
def test_vit_assemble(B, scale):
    ops = _ops()
    L, Lp, C = 257, 264, 1024
    patches = _randn(B * (L - 1), C, seed=B, dtype=BF16)
    cls = _randn(C, seed=10)
    pos = _randn(L, C, seed=11, scale=0.3)
    ts = None
    if scale != "none":
        ts = torch.rand(B, L, generator=_gen(12), device=DEV) + 0.5
        if scale == "zeros":
            ts[:, ::7] = 0.0
    out = ops.vit_assemble(patches, cls, pos, B, L, Lp, tok_scale=ts)
    v = torch.cat([cls.expand(B, 1, C), patches.float().view(B, L - 1, C)], 1) + pos[:L]
    if ts is not None:
        v = v * ts[:, :, None]
    ref = torch.zeros(B, Lp, C, dtype=BF16, device=DEV)
    ref[:, :L] = v.to(BF16)
    check_bitwise(out, ref, f"vit_assemble B{B} tok_scale {scale}")


@pytest.mark.parametrize("L,Lp,idx", [(77, 80, (6, 13, 76)), (77, 80, None), (257, 264, (6, 130, 256)), (257, 264, None)])
@pytest.mark.parametrize("soft", [False, True])
def test_scale_by_row_norm(L, Lp, idx, soft):
    ops = _ops()
    B, C = 3, 768
    z = _randn(B, Lp, C, seed=L + Lp)
    z = (z * (1.0 + (torch.arange(Lp, device=DEV) % 2))[None, :, None]).to(BF16)    # neighbouring rows' norms differ by 2x
    it = None if idx is None else torch.tensor(idx, dtype=torch.int32, device=DEV)
    rs = torch.rand(B, L, generator=_gen(5), device=DEV) + 0.5 if soft else None
    out = ops.scale_by_row_norm(z, L, idx=it, row_scale=rs)
    rows = [0] * B if idx is None else list(idx)
    zd = z.double()
    nrm = torch.stack([zd[b, rows[b]].norm() for b in range(B)])
    ref = zd[:, :L] / nrm[:, None, None]
    if soft:
        ref = ref * rs.double()[:, :, None]
    D = math.ceil(C / 256) + 13
    check_bound(out, ref, (D / 2 + 4) * U * ref.abs(), f"scale_by_row_norm L{L} idx {idx} row_scale {'soft' if soft else None}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_clip_to_u8_hwc, vdb_resample_h_u8, vdb_resample_v_crop_norm
# ---------------------------------------------------------------------------------------------------------------------------
def test_clip_to_u8_hwc_truncates_like_topilimage():
    ops = _ops()
    k = torch.arange(256, dtype=torch.float32) / 255.0
    vals = torch.cat([k, torch.nextafter(k, torch.tensor(-1.0)), torch.nextafter(k, torch.tensor(2.0)),
                      torch.tensor([-1.0, -1e-30, -0.0, 1.0000001, 1.5, 3e38])])
    n, H, W = 2, 7, (3 * vals.numel() + 13) // 14
    x = torch.rand(n * 3 * H * W, generator=torch.Generator().manual_seed(1))
    x[:vals.numel()] = vals
    x[-vals.numel():] = vals.flip(0)
    x = x.view(n, 3, H, W).to(DEV)
    out = ops.to_uint8_hwc(x)
    ref = (x.clamp(0, 1) * 255).byte().permute(0, 2, 3, 1).contiguous()
    check_bitwise(out, ref, "clip_to_u8_hwc")


RS_SHAPES = [  # (n, H, W): strong downscales (11- and 21-tap kernels), upscales on both axes, crop only, odd crop offsets
    (1, 512, 2048), (1, 1024, 1024), (3, 60, 50), (3, 224, 302), (1, 100, 130),
]


def _pre_tables(H, W, size=224):
    from lib.model_zoo.clip import CLIPImageContextEncoder as E
    nw, nh = (size, int(size * H / W)) if W <= H else (int(size * W / H), size)
    return nw, nh, (E.pil_bicubic_coeffs(W, nw) if nw != W else None), (E.pil_bicubic_coeffs(H, nh) if nh != H else None)


@pytest.mark.parametrize("n,H,W", RS_SHAPES)
def test_clip_preprocess_passes_are_bit_exact_with_pillow(n, H, W):
    from oracle import pil_resample as pr
    ops, lib = _ops(), _ops().lib
    size = 224
    nw, nh, th, tv = _pre_tables(H, W, size)
    imgs = torch.rand(n, 3, H, W, generator=torch.Generator().manual_seed(H * 7 + W))
    x = imgs.to(DEV)
    u8 = ops.to_uint8_hwc(x)
    u8_ref = (imgs.numpy().clip(0.0, 1.0).astype(np.float32) * np.float32(255)).astype(np.uint8).transpose(0, 2, 3, 1)
    check_bitwise(u8, torch.from_numpy(np.ascontiguousarray(u8_ref)), f"clip_to_u8 {n}x{H}x{W}")
    mid_ref = u8_ref
    if th is not None:
        hb, hk = (torch.from_numpy(a).to(DEV) for a in th)
        mid = torch.empty(n, H, nw, 3, dtype=torch.uint8, device=DEV)
        ops.check(lib.vdb_resample_h_u8(u8.data_ptr(), n, H, W, nw, hb.data_ptr(), hk.data_ptr(), hk.shape[1], mid.data_ptr(),
                                        ops._stream()), "resample_h_u8")
        mid_ref = np.stack([pr.resample_pass(im, *pr.coefficients(W, nw), axis=1) for im in u8_ref])
        print(f"resample_h {W} -> {nw}: {hk.shape[1]} taps")
        check_bitwise(mid, torch.from_numpy(mid_ref), f"resample_h_u8 {n}x{H}x{W}")
        u8_mid = mid
    else:
        u8_mid = u8
    top, left = (nh - size) // 2, (nw - size) // 2
    col_ref = mid_ref
    if tv is not None:
        col_ref = np.stack([pr.resample_pass(im, *pr.coefficients(H, nh), axis=0) for im in mid_ref])
        print(f"resample_v {H} -> {nh}: {tv[1].shape[1]} taps")
    crop = col_ref[:, top:top + size, left:left + size].astype(np.float32) / np.float32(255.0)
    crop = (crop - np.asarray(pr.IMAGE_MEAN, dtype=np.float32)) / np.asarray(pr.IMAGE_STD, dtype=np.float32)
    ref = torch.from_numpy(np.ascontiguousarray(crop.transpose(0, 3, 1, 2)))
    out = torch.empty(n, 3, size, size, dtype=torch.float32, device=DEV)
    vb, vk = (None, None) if tv is None else (torch.from_numpy(a).to(DEV) for a in tv)
    import ctypes
    m3, s3 = (ctypes.c_float * 3)(*pr.IMAGE_MEAN), (ctypes.c_float * 3)(*pr.IMAGE_STD)
    ops.check(lib.vdb_resample_v_crop_norm(u8_mid.data_ptr(), n, H, nw, 0 if vb is None else vb.data_ptr(),
                                           0 if vk is None else vk.data_ptr(), 0 if vk is None else vk.shape[1], top, left, size,
                                           m3, s3, out.data_ptr(), ops._stream()), "resample_v_crop_norm")
    print(f"crop offsets top {top} left {left}")
    check_bitwise(out, ref, f"resample_v_crop_norm {n}x{H}x{W}")
    tables = {"nw": nw, "nh": nh, "h": None if th is None else tuple(torch.from_numpy(a).to(DEV) for a in th),
              "v": None if tv is None else tuple(torch.from_numpy(a).to(DEV) for a in tv)}
    chain = ops.clip_preprocess_device(x, tables, size, pr.IMAGE_MEAN, pr.IMAGE_STD)
    check_bitwise(chain, torch.from_numpy(pr.clip_preprocess(imgs.numpy(), size)), f"clip_preprocess chain {n}x{H}x{W}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_pointwise_small, vdb_gaussian_sample
# ---------------------------------------------------------------------------------------------------------------------------
PW_CASES = [(8, 8, 1.0), (4, 4, 1 / 0.18215), (3, 5, 1.0), (1, 1, 1.0), (8, 1, 1.0)]


@pytest.mark.parametrize("cin,cout,pre", PW_CASES)
@pytest.mark.parametrize("with_bias", [False, True])
def test_pointwise_small(cin, cout, pre, with_bias):
    ops = _ops()
    w = _randn(cout, cin, seed=cin * 10 + cout, scale=0.5)
    b = _randn(cout, seed=3) if with_bias else None
    pre32 = _f32(pre)
    for npix in (1, 7, 64 * 64 * 4, ew_limit() + 1):
        x = _randn(npix, cin, seed=npix, scale=2.0)
        out = ops.pointwise_small(x, w, b, pre_mul=pre)
        xp = x.double() * pre32
        bd = b.double() if with_bias else torch.zeros(cout, dtype=torch.float64, device=DEV)
        ref = xp @ w.double().t() + bd
        bound = (cin + 2) * U * (xp.abs() @ w.double().abs().t() + bd.abs())
        check_bound(out, ref, bound, f"pointwise_small {cin}->{cout} pre {pre32:.6g} bias {int(with_bias)} npix {npix}")


@pytest.mark.parametrize("with_noise", [True, False])
@pytest.mark.parametrize("post", [0.18215, 1.0])
def test_gaussian_sample(with_noise, post):
    ops = _ops()
    C, npix = 4, 4096 + 3
    mom = torch.empty(npix, 2 * C, device=DEV)
    mom[:, :C] = _randn(npix, C, seed=1, scale=2.0)
    lv = torch.rand(npix, C, generator=_gen(2), device=DEV) * 70 - 40                 # logvar across [-40, 30]
    lv[:8] = torch.tensor([-30.0, 20.0, -40.0, 30.0, 19.5, 19.0, 20.5, -29.5], device=DEV)[:, None]
    mom[:, C:] = lv
    noise = _randn(npix, C, seed=3) if with_noise else None
    out = ops.gaussian_sample(mom, noise, post_mul=post)
    p32 = _f32(post)
    m = mom[:, :C].double()
    if with_noise:
        sn = torch.exp(0.5 * mom[:, C:].double().clamp(-30, 20)) * noise.double()
    else:
        sn = torch.zeros_like(m)
    ref = (m + sn) * p32
    bound = abs(p32) * (7 * U * sn.abs() + 2 * U * m.abs())
    check_bound(out, ref, bound, f"gaussian_sample noise {int(with_noise)} post {post}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_im2col3x3_small, vdb_permute_f32, vdb_upsample2x_nhwc
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1, 1), (1, 7), (5, 3), (64, 64), (512, 512)])
@pytest.mark.parametrize("cin", [3, 4])
@pytest.mark.parametrize("B", [1, 3])
def test_im2col3x3_small(H, W, cin, B):
    ops = _ops()
    kpad = 64
    x = _randn(B, H, W, cin, seed=H * W + cin)
    for s, t in ((1.0, 0.0), (2.0, -1.0)):
        out = ops.im2col3x3_small(x, kpad=kpad, in_scale=s, in_shift=t)
        xt = x.permute(0, 3, 1, 2) * s + t
        unf = F.unfold(xt, 3, padding=1).view(B, cin, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 9 * cin)
        ref = torch.zeros(B * H * W, kpad, dtype=BF16, device=DEV)
        ref[:, :9 * cin] = unf.to(BF16)
        check_bitwise(out, ref, f"im2col3x3_small B{B} {H}x{W} Cin{cin} ({s}, {t})")


PERM_CASES = [(1, 3, 37, 53), (5, 4, 37, 53), (5, 8, 37, 53), (1, 8, 37, 53), (1, 3, 512, 2048)]


@pytest.mark.parametrize("B,C,H,W", PERM_CASES)
def test_permute(B, C, H, W):
    ops = _ops()
    x = _randn(B, C, H, W, seed=B * C + H, scale=1.5)
    if B * C * H * W > 16 * _sms() * 256:
        print(f"permute {B}x{C}x{H}x{W}: grid-stride")
    for mul, add in ((1.0, 0.0), (2.0, -1.0)):
        check_bitwise(ops.nchw_to_nhwc(x, mul=mul, add=add), (x * mul + add).permute(0, 2, 3, 1).contiguous(),
                      f"nchw_to_nhwc {B}x{C}x{H}x{W} ({mul}, {add})")
    xh = x.permute(0, 2, 3, 1).contiguous()
    check_bitwise(ops.nhwc_to_nchw(xh), x, f"nhwc_to_nchw {B}x{C}x{H}x{W}")
    check_bitwise(ops.nhwc_to_nchw(xh, mul=0.5, add=0.5, clamp01=True), torch.clamp((x + 1) / 2, 0, 1),
                  f"nhwc_to_nchw decode {B}x{C}x{H}x{W}")


@pytest.mark.parametrize("C", [8, 520])
def test_upsample2x(C):
    ops = _ops()
    x = _randn(3, 5, 7, C, seed=C, dtype=BF16)
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    check_bitwise(ops.upsample2x(x), ref, f"upsample2x C{C}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_cast_f32_bf16, vdb_cast_bf16_f32
# ---------------------------------------------------------------------------------------------------------------------------
def _bits_f32(v):
    return torch.tensor(np.array(v, dtype=np.uint32).view(np.int32)).view(torch.float32)


def _bf16_rne(x):
    """c10's float -> bfloat16 (round to nearest even on the bit pattern, NaN -> 0x7FC0), restated in integers."""
    u = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    r = torch.where((u & 0x7FFFFFFF) > 0x7F800000, torch.full_like(r, 0x7FC0), r)
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16).view(BF16)


def test_cast_f32_bf16():
    ops = _ops()
    g = torch.Generator().manual_seed(4)
    n = ew_limit() + 1001
    bits = torch.randint(-2 ** 31, 2 ** 31, (n,), dtype=torch.int64, generator=g).to(torch.int32)
    x = bits.view(torch.float32).clone()
    hi = torch.randint(0, 0x7F80, (512,), generator=g, dtype=torch.int64)
    hi = torch.cat([hi & ~1, hi | 1])                                              # even and odd bf16 mantissas
    ties = (hi << 16) | 0x8000                                                     # exactly halfway
    near = torch.cat([(hi << 16) | 0x7FFF, (hi << 16) | 0x8001])
    special = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001, 0x00000001, 0x80000001,
               0x00008000, 0x00018000, 0x007FFFFF, 0x807F8000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF]
    spec = torch.cat([ties, ties | (1 << 31), near, torch.tensor(special, dtype=torch.int64)])
    x[:spec.numel()] = _bits_f32(spec.numpy().astype(np.uint32))
    x[-spec.numel():] = _bits_f32(spec.numpy().astype(np.uint32))
    xd = x.to(DEV)
    out = ops.to_bf16(xd)
    check_bitwise(out, _bf16_rne(x), f"cast_f32_bf16 n {n}")
    check_bitwise(out, xd.to(BF16), f"cast_f32_bf16 n {n} vs torch")
    assert out[spec.numel() - 4].view(torch.int16).item() == 0x7F80, "max finite fp32 must round to +inf"


def test_cast_bf16_f32():
    ops = _ops()
    n = ew_limit() + 1001
    bits = torch.randint(-2 ** 15, 2 ** 15, (n,), dtype=torch.int64, generator=torch.Generator().manual_seed(5)).to(torch.int16)
    x = bits.view(BF16)
    check_bitwise(ops.to_f32(x.to(DEV)), x.float(), f"cast_bf16_f32 n {n}")


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_mask_to_latent
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("H8,W8", [(8, 8), (64, 512), (512, 4096)])
def test_mask_to_latent(n, H8, W8):
    ops = _ops()
    m = (torch.rand(n, 1, H8, W8, generator=_gen(H8 + W8 + n), device=DEV) * 4).floor() / 3       # many ties
    m[-1, 0, -8:, -8:] = 0.25                                       # a cell of equal values
    m[0, 0, 3, 5] = math.nan                                        # a NaN inside the first cell, after its first element
    if W8 > 8:
        m[0, 0, 0, 8] = math.nan                                    # a NaN as the first element of a cell
    out = ops.mask_to_latent(m)
    check_bitwise(out, F.max_pool2d(m, 8), f"mask_to_latent n{n} {H8}x{W8}")
    assert torch.isnan(out[0, 0, 0, 0])


# ---------------------------------------------------------------------------------------------------------------------------
# vdb_axpby_f32, vdb_lincomb4_f32
# ---------------------------------------------------------------------------------------------------------------------------
def test_axpby():
    ops = _ops()
    a, b = _f32(math.sqrt(0.3)), _f32(math.sqrt(0.7))
    for n in (1, 5, 66, ew_limit() + 1):
        x, z = _randn(n, seed=n), _randn(n, seed=n + 1)
        check_bitwise(ops.axpby(x, z, a, b), x * a + z * b, f"axpby n {n}")


PLMS = [(0.5, 0.5), (1.5, -0.5), (23. / 12, -16. / 12, 5. / 12), (55. / 24, -59. / 24, 37. / 24, -9. / 24)]


@pytest.mark.parametrize("cs", [(1.0,)] + PLMS, ids=["1", "2", "2b", "3", "4"])
def test_lincomb4(cs):
    ops = _ops()
    for n in (5, 4 * 64 * 64 * 2 + 3, ew_limit() + 1):
        xs = [_randn(n, seed=10 * i + n) for i in range(len(cs))]
        out = ops.lincomb4(xs, cs)
        t = [_f32(c) * x.double() for c, x in zip(cs, xs)]
        S, bound = torch.zeros_like(t[0]), torch.zeros_like(t[0])
        for i, ti in enumerate(t):
            S = S + ti
            bound = bound + U * S.abs() + (U * ti.abs() if i else 0)
        check_bound(out, S, bound, f"lincomb4 {len(cs)} terms n {n}")


# ---------------------------------------------------------------------------------------------------------------------------
# Shape checks: every wrapper refuses a short or mismatched buffer before it launches anything
# ---------------------------------------------------------------------------------------------------------------------------
def _refusals():
    f32 = dict(dtype=torch.float32, device=DEV)
    z = lambda *s: torch.zeros(*s, **f32)
    zb = lambda *s: torch.zeros(*s, dtype=BF16, device=DEV)
    ts = torch.zeros(4, dtype=torch.int64, device=DEV)
    return {
        "linear_small-w-K": lambda o: o.linear_small(z(2, 64), zb(32, 56)),
        "linear_small-bias": lambda o: o.linear_small(z(2, 64), zb(32, 64), z(31)),
        "linear_small-out": lambda o: o.linear_small(z(2, 64), zb(32, 64), out=z(2, 31)),
        "softmax_rows-out": lambda o: o.softmax_rows(zb(8, 64), out=zb(8, 32)),
        "axpby-z": lambda o: o.axpby(z(100), z(99), 1.0, 1.0),
        "axpby-out": lambda o: o.axpby(z(100), z(100), 1.0, 1.0, out=z(50)),
        "lincomb4-xs": lambda o: o.lincomb4([z(100), z(100), z(64)], [1.0, 1.0, 1.0]),
        "lincomb4-out": lambda o: o.lincomb4([z(100), z(100)], [1.0, 1.0], out=z(10)),
        "pointwise_small-x": lambda o: o.pointwise_small(z(16, 4), z(4, 8)),
        "pointwise_small-bias": lambda o: o.pointwise_small(z(16, 8), z(4, 8), z(8)),
        "pointwise_small-out": lambda o: o.pointwise_small(z(16, 8), z(4, 8), out=z(16, 3)),
        "gaussian_sample-noise": lambda o: o.gaussian_sample(z(16, 8), z(16, 3)),
        "gaussian_sample-odd": lambda o: o.gaussian_sample(z(16, 7)),
        "gaussian_sample-out": lambda o: o.gaussian_sample(z(16, 8), out=z(16, 2)),
        "timestep_embedding-out": lambda o: o.timestep_embedding(ts, 320, out=z(4, 160)),
        "to_bf16-out": lambda o: o.to_bf16(z(100), out=zb(99)),
        "to_f32-out": lambda o: o.to_f32(zb(100), out=z(99)),
        "scale_by_row_norm-idx": lambda o: o.scale_by_row_norm(zb(3, 80, 64), 77, idx=torch.zeros(2, dtype=torch.int32, device=DEV)),
        "scale_by_row_norm-row_scale": lambda o: o.scale_by_row_norm(zb(3, 80, 64), 77, row_scale=z(3, 76)),
        "vit_assemble-patches": lambda o: o.vit_assemble(zb(2 * 255, 64), z(64), z(257, 64), 2, 257, 264),
        "vit_assemble-cls": lambda o: o.vit_assemble(zb(2 * 256, 64), z(63), z(257, 64), 2, 257, 264),
        "vit_assemble-pos": lambda o: o.vit_assemble(zb(2 * 256, 64), z(64), z(256, 64), 2, 257, 264),
        "vit_assemble-tok_scale": lambda o: o.vit_assemble(zb(2 * 256, 64), z(64), z(257, 64), 2, 257, 264, tok_scale=z(2, 256)),
        "clip_text_embed-pos": lambda o: o.clip_text_embed(torch.zeros(2, 77, dtype=torch.int64, device=DEV), z(100, 64), z(76, 64), 80),
    }


REFUSALS = ["linear_small-w-K", "linear_small-bias", "linear_small-out", "softmax_rows-out", "axpby-z", "axpby-out", "lincomb4-xs",
            "lincomb4-out", "pointwise_small-x", "pointwise_small-bias", "pointwise_small-out", "gaussian_sample-noise",
            "gaussian_sample-odd", "gaussian_sample-out", "timestep_embedding-out", "to_bf16-out", "to_f32-out",
            "scale_by_row_norm-idx", "scale_by_row_norm-row_scale", "vit_assemble-patches", "vit_assemble-cls", "vit_assemble-pos",
            "vit_assemble-tok_scale", "clip_text_embed-pos"]


@pytest.mark.parametrize("case", REFUSALS)
def test_wrapper_refuses_mismatched_buffers_before_launching(case):
    ops = _ops()
    call = _refusals()[case]
    torch.cuda.synchronize()
    before = ops.launch_count()
    with pytest.raises(ValueError):
        call(ops)
    assert ops.launch_count() == before, f"{case}: a kernel was launched before the refusal"
