"""Per-kernel numerics: every vdb200 kernel against a plain torch fp32 restatement of the same op
(the reference's own arithmetic for that call site), on bf16-rounded inputs.

Tolerances: bf16 tensor-core kernels  max|err| <= 2e-2 * max|ref| and cosine >= 0.999;
fp32 elementwise kernels bit-exact or <= 1e-6 relative as stated per test.  test_igemm_coverage_gpu.py checks every
implicit-GEMM instantiation per element against fp64.
"""
import math

import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from vdb200 import ops
    return ops


def rnd(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def assert_close(out, ref, tol=2e-2, cos_min=0.999, what=""):
    out = out.float().flatten()
    ref = ref.float().flatten()
    assert torch.isfinite(out).all(), f"{what}: non-finite output"
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-12
    cos = F.cosine_similarity(out, ref, dim=0).item()
    assert err <= tol * scale and cos >= cos_min, f"{what}: max err {err:.4g} vs scale {scale:.4g}, cos {cos:.6f}"


# ----------------------------------------------------------------------------------------------
def test_ddim_cfg_step_bit_exact():
    ops = _ops()
    n = (4, 64, 64, 4)
    eu, ec, x = (rnd(*n, seed=s, dtype=torch.float32) for s in (1, 2, 3))
    a_t, a_prev, sigma = 0.5312, 0.6123, 0.0
    coef = torch.tensor([[a_t, a_prev, sigma, math.sqrt(1 - a_t)]], dtype=torch.float32, device=DEV)
    p0 = torch.empty_like(x)
    xp, _ = ops.ddim_cfg_step(eu, ec, x, coef, 7.5, pred_x0=p0)
    # reference op order of ddim.py:150,165-170 (separate fp32 ATen ops)
    e = eu + 7.5 * (ec - eu)
    c = coef[0]
    px0 = (x - c[3] * e) / c[0].sqrt()
    d = (1.0 - c[1] - c[2] ** 2).sqrt() * e
    ref = c[1].sqrt() * px0 + d + c[2] * torch.zeros_like(x) * 1.0
    assert torch.equal(p0, px0)
    assert torch.equal(xp, ref)


def test_ddim_cfg_step_table_and_noise():
    ops = _ops()
    x, ec, nz = (rnd(2, 33, seed=s, dtype=torch.float32) for s in (1, 2, 3))  # n = 66: tail path
    coef = torch.tensor([[0.9, 0.95, 0.0, 0.3], [0.4, 0.5, 0.2, 0.77]], dtype=torch.float32, device=DEV)
    idx = torch.tensor([1], dtype=torch.int32, device=DEV)
    xp, _ = ops.ddim_cfg_step(None, ec, x, coef, 1.0, noise=nz, temperature=0.7, step_idx=idx)
    c = coef[1]
    px0 = (x - c[3] * ec) / c[0].sqrt()
    ref = c[1].sqrt() * px0 + (1.0 - c[1] - c[2] ** 2).sqrt() * ec + c[2] * nz * 0.7
    assert torch.equal(xp, ref)
    ops.add_int(idx, -1)
    assert idx.item() == 0


GEMM_CASES = [
    # M, N, K, bias, resid, act, bn, ksplit, f32out
    (128, 64, 64, False, False, 0, 0, 1, False),
    (256, 160, 320, True, False, 0, 0, 1, False),
    (1000, 320, 320, True, True, 0, 0, 1, False),
    (4096, 1280, 640, True, True, 0, 0, 1, False),
    (77, 768, 768, True, False, 3, 0, 1, False),
    (300, 256, 128, True, False, 1, 128, 1, False),
    (512, 1280, 2880, True, True, 0, 0, 0, False),     # auto BN and split-K (132 SMs: the tile-width model picks BN 64, no split)
    (512, 1280, 11520, True, True, 0, 0, 8, False),    # forced split-K
    (640, 200, 192, True, False, 2, 0, 1, True),       # fp32 out, N tail
    (8192, 320, 1280, False, True, 0, 160, 1, False),
    (20000, 640, 640, True, False, 0, 0, 1, False),    # many tiles per CTA (persistent loop)
]


@pytest.mark.parametrize("M,N,K,bias,resid,act,bn,ksplit,f32", GEMM_CASES)
def test_gemm(M, N, K, bias, resid, act, bn, ksplit, f32):
    ops = _ops()
    a = rnd(M, K, seed=1)
    w = rnd(N, K, seed=2, scale=K ** -0.5)
    b = rnd(N, seed=3, dtype=torch.float32) if bias else None
    r = rnd(M, N, seed=4) if resid else None
    out = ops.gemm(a, w, bias=b, resid=r, act=act, bn=bn, ksplit=ksplit,
                   out_dtype=torch.float32 if f32 else torch.bfloat16)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b
    ref = {0: lambda t: t, 1: F.silu, 2: F.gelu, 3: lambda t: t * torch.sigmoid(1.702 * t)}[act](ref)
    if resid:
        ref = ref + r.float()
    assert_close(out, ref, what=f"gemm {M}x{N}x{K}")


def test_gemm_two_source_and_batched_bias():
    ops = _ops()
    M, K1, K2, N, B = 512, 640, 320, 320, 4
    a1, a2 = rnd(M, K1, seed=1), rnd(M, K2, seed=2)
    w = rnd(N, K1 + K2, seed=3, scale=(K1 + K2) ** -0.5)
    bias = rnd(B, N, seed=4, dtype=torch.float32)
    out = ops.gemm(a1, w, a2=a2, bias=bias, bias_bstride=N, rows_per_batch=M // B)
    ref = torch.cat([a1, a2], 1).float() @ w.float().t() + bias.repeat_interleave(M // B, 0)
    assert_close(out, ref, what="gemm two-source")


def pack_geglu(w, b, bn=256):
    """rows [0,4C) value, [4C,8C) gate -> per 256-col tile: 128 value rows then their 128 gate rows"""
    n2 = w.shape[0] // 2
    half = bn // 2
    idx = []
    for t in range(n2 // half):
        idx += list(range(t * half, (t + 1) * half)) + list(range(n2 + t * half, n2 + (t + 1) * half))
    idx = torch.tensor(idx, device=w.device)
    return w[idx].contiguous(), (b[idx].contiguous() if b is not None else None)


@pytest.mark.parametrize("M,C", [(256, 320), (1024, 640)])
def test_gemm_geglu(M, C):
    ops = _ops()
    x = rnd(M, C, seed=1)
    w = rnd(8 * C, C, seed=2, scale=C ** -0.5)
    b = rnd(8 * C, seed=3, dtype=torch.float32)
    wp, bp = pack_geglu(w, b)
    out = ops.gemm(x, wp, bias=bp, act=ops.ACT_GEGLU)
    h = x.float() @ w.float().t() + b
    val, gate = h.chunk(2, dim=-1)
    ref = val * F.gelu(gate)
    assert out.shape == (M, 4 * C)
    assert_close(out, ref, what="geglu")


# ---- LayerNorm folded into the GEMMs (vdb_gemm_ln_bf16) ------------------------------------------------------------------
def _chunk_stats(x, width=32):
    """[M, C] fp32 -> [C/width, M, 2] partial (sum, sum of squares) over column ranges: the kind of table a producer GEMM writes"""
    M, C = x.shape
    xc = x.view(M, C // width, width)
    return torch.stack([xc.sum(-1), (xc * xc).sum(-1)], -1).permute(1, 0, 2).contiguous()


def _ln(x, C, width=32):
    st = _chunk_stats(x.float(), width)
    return _ops().LnFold(st, st.shape[0], C, 1e-5)


def _fold(w, b, gamma, beta):
    wg = (w.float() * gamma[None, :]).to(torch.bfloat16).contiguous()
    c = w.float() @ beta + (b if b is not None else 0)
    return wg, wg.float().sum(1).contiguous(), c.contiguous()


@pytest.mark.parametrize("M,N,K,resid,bn", [(1024, 320, 320, True, 0), (520, 640, 1280, True, 0), (4096, 320, 320, False, 160),
                                            (300, 1280, 512, True, 64)])
def test_gemm_ln_producer_writes_chunk_statistics(M, N, K, resid, bn):
    ops = _ops()
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=K ** -0.5)
    b = rnd(N, seed=3, dtype=torch.float32)
    r = rnd(M, N, seed=4) if resid else None
    st = ops.ln_stats_buffer(M, N, a.device)
    st.fill_(float("nan"))
    out, parts = ops.gemm_ln(a, w, bias=b, resid=r, stats_out=st, bn=bn)
    ref = a.float() @ w.float().t() + b + (r.float() if resid else 0)
    assert_close(out, ref, what=f"gemm_ln producer {M}x{N}x{K}")
    assert 2 <= parts <= st.shape[0] and torch.isfinite(st[:parts]).all()
    tot = st[:parts].sum(0)                                       # [M, 2]: the partials add up to the row sums
    ref_tot = torch.stack([ref.sum(1), (ref * ref).sum(1)], -1)
    err = (tot - ref_tot).abs().max().item()
    assert err <= 2e-3 * ref_tot.abs().max().item() + 1e-3, f"row statistics off by {err}"


@pytest.mark.parametrize("M,N,C,bias,mean", [(1024, 1024, 320, False, 0.0), (2048, 512, 640, True, 1.5), (384, 2048, 1280, True, -0.7),
                                             (100, 320, 320, True, 4.0)])
def test_gemm_ln_consumer_rows(M, N, C, bias, mean):
    """Linear(LayerNorm(x)) from the raw x + per-chunk statistics; `mean` shifts the rows (the rank-1 term must cancel it)"""
    ops = _ops()
    x = (rnd(M, C, seed=1).float() * 1.3 + mean).to(torch.bfloat16)
    w0 = rnd(N, C, seed=2, scale=C ** -0.5)
    b0 = rnd(N, seed=3, dtype=torch.float32) if bias else None
    gamma = 1.0 + 0.3 * rnd(C, seed=4, dtype=torch.float32)
    beta = 0.2 * rnd(C, seed=5, dtype=torch.float32)
    wg, s, c = _fold(w0, b0, gamma, beta)
    out = ops.gemm_ln(x, wg, bias=c, ln=_ln(x, C, 32 if C > 320 else 160), colsum=s)     # 2 .. 40 partials per row
    ref = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w0.float().t() + (b0 if bias else 0)
    assert_close(out, ref, what=f"gemm_ln rows {M}x{N}x{C} mean {mean}")


@pytest.mark.parametrize("T,R,C", [(4096, 384, 320), (992, 384, 640), (256, 640, 1280)])
def test_gemm_ln_consumer_columns(T, R, C):
    """the transposed projection: out^T [R, T] = W0 LayerNorm(x)^T, statistics per output COLUMN (token)"""
    ops = _ops()
    x = (rnd(T, C, seed=1).float() + 0.8).to(torch.bfloat16)
    w0 = rnd(R, C, seed=2, scale=C ** -0.5)
    gamma = 1.0 + 0.3 * rnd(C, seed=4, dtype=torch.float32)
    beta = 0.2 * rnd(C, seed=5, dtype=torch.float32)
    wg, s, c = _fold(w0, None, gamma, beta)
    out = ops.gemm_ln(wg, x, ln=_ln(x, C, 64), colsum=s, on_cols=True, rowbias=c)
    ref = w0.float() @ F.layer_norm(x.float(), (C,), gamma, beta, 1e-5).t()
    assert out.shape == (R, T)
    assert_close(out, ref, what=f"gemm_ln columns {R}x{T}x{C}")


@pytest.mark.parametrize("M,C", [(512, 320), (1024, 640)])
def test_gemm_ln_consumer_geglu(M, C):
    ops = _ops()
    x = (rnd(M, C, seed=1).float() * 0.9 - 0.4).to(torch.bfloat16)
    w0 = rnd(8 * C, C, seed=2, scale=C ** -0.5)
    b0 = rnd(8 * C, seed=3, dtype=torch.float32)
    gamma = 1.0 + 0.3 * rnd(C, seed=4, dtype=torch.float32)
    beta = 0.2 * rnd(C, seed=5, dtype=torch.float32)
    wg, s, c = _fold(w0, b0, gamma, beta)
    wp, cp = pack_geglu(wg, c)
    _, sp = pack_geglu(wg, s)
    out = ops.gemm_ln(x, wp, bias=cp, act=ops.ACT_GEGLU, ln=_ln(x, C, 80), colsum=sp)
    h = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w0.float().t() + b0
    val, gate = h.chunk(2, dim=-1)
    assert out.shape == (M, 4 * C)
    assert_close(out, val * F.gelu(gate), what="gemm_ln geglu")


def test_gemm_ln_rejects_what_the_tma_store_epilogue_cannot_do():
    from vdb200._lib import VdbError
    ops = _ops()
    x, w = rnd(1000, 320, seed=1), rnd(384, 320, seed=2)
    s = torch.zeros(384, device=DEV)
    with pytest.raises(VdbError):        # 1000 output columns: not a multiple of 32
        ops.gemm_ln(w, x, ln=_ln(x, 320), colsum=s, on_cols=True)
    with pytest.raises(VdbError):        # neither consumer nor producer
        ops.gemm_ln(x, w)


def test_gemm_ln_producer_feeds_consumer():
    """the real chain: producer GEMM (+resid) writes the statistics of ITS bf16 output rows, the consumer normalises with them"""
    ops = _ops()
    M, C, N = 2048, 320, 1024
    a, w = rnd(M, C, seed=1), rnd(C, C, seed=2, scale=C ** -0.5)
    r = rnd(M, C, seed=3)
    st = ops.ln_stats_buffer(M, C, a.device)
    x, parts = ops.gemm_ln(a, w, resid=r, stats_out=st)
    w0 = rnd(N, C, seed=4, scale=C ** -0.5)
    gamma = 1.0 + 0.3 * rnd(C, seed=5, dtype=torch.float32)
    beta = 0.2 * rnd(C, seed=6, dtype=torch.float32)
    wg, s, c = _fold(w0, None, gamma, beta)
    out = ops.gemm_ln(x, wg, bias=c, ln=ops.LnFold(st, parts, C, 1e-5), colsum=s)
    ref = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w0.float().t()
    assert_close(out, ref, what="gemm_ln chain")
    via_kernel = ops.gemm(ops.layernorm(x, gamma, beta, eps=1e-5), w0)
    assert_close(out, via_kernel.float(), what="gemm_ln chain vs LayerNorm kernel + GEMM")


@pytest.mark.parametrize("B,H,W,C,N", [(2, 16, 16, 64, 64), (8, 32, 32, 640, 640), (1, 24, 40, 128, 192), (3, 8, 8, 128, 320)])
def test_folded_upsample_conv_direct_store_equals_interleave_pass(B, H, W, C, N):
    """nearest-2x upsample + 3x3 conv as four parity convs on the source: conv modes 7..10 store every parity straight into the
    [B,2H,2W,N] result through the output tensor map, and the result matches torch's upsample + conv2d on the bf16-rounded
    operands (Upsample.forward, openaimodel.py:107-117)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "versatile-diffusion_b200"))
    from lib.model_zoo.diffusion_utils import fold_upsample_conv3x3
    ops = _ops()
    g = torch.Generator().manual_seed(H * 7 + C)
    x = torch.randn(B, H, W, C, generator=g).to(torch.bfloat16).to(DEV)
    w = torch.randn(N, C, 3, 3, generator=g) * 0.05
    b = torch.randn(N, generator=g).to(DEV)
    wf = fold_upsample_conv3x3(w).to(DEV)
    direct = ops.upsample2x_conv3x3_folded(x, wf, bias=b)
    assert direct.shape == (B, 2 * H, 2 * W, N)
    ref = F.conv2d(F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest"),
                   w.to(torch.bfloat16).float().to(DEV), b, padding=1).permute(0, 2, 3, 1)
    assert_close(direct, ref, tol=3e-2, what=f"folded upsample conv {B}x{H}x{W} {C}->{N}")


def pack_conv_w(w, skip_ws=()):
    """[N,C,3,3] -> [N, (ky,kx,c)] (+ 1x1 skip columns)"""
    cols = [w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)]
    cols += [s.reshape(s.shape[0], -1) for s in skip_ws]
    return torch.cat(cols, 1).contiguous()


CONV_CASES = [
    # B, H, W, C, N, mode
    (2, 64, 64, 64, 128, 0),
    (2, 16, 16, 128, 160, 0),
    (3, 8, 8, 64, 64, 0),
    (1, 32, 32, 320, 320, 0),
    (2, 32, 32, 64, 64, 1),
    (3, 16, 16, 128, 128, 1),
    (2, 32, 32, 64, 64, 2),
    (1, 256, 256, 64, 64, 0),
    (2, 8, 8, 1280, 1280, 0),   # split-K regime
]


@pytest.mark.parametrize("B,H,W,C,N,mode", CONV_CASES)
def test_conv3x3(B, H, W, C, N, mode):
    ops = _ops()
    x = rnd(B, H, W, C, seed=1)
    w = rnd(N, C, 3, 3, seed=2, scale=(9 * C) ** -0.5)
    bias = rnd(N, seed=3, dtype=torch.float32)
    out = ops.conv3x3(x, pack_conv_w(w), bias=bias, mode=mode)
    xin = x.float().permute(0, 3, 1, 2)
    if mode == 0:
        ref = F.conv2d(xin, w.float(), bias, padding=1)
    elif mode == 1:
        ref = F.conv2d(xin, w.float(), bias, stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(xin, (0, 1, 0, 1)), w.float(), bias, stride=2)
    assert_close(out, ref.permute(0, 2, 3, 1), what=f"conv {B}x{H}x{W}x{C}->{N} mode {mode}")


def test_conv3x3_resblock_tail():
    """conv2 of a channel-changing ResBlock: 3x3 conv + 1x1 skip over cat(h, skip) + per-batch bias + residual"""
    ops = _ops()
    B, H, W, C, N, C1, C2 = 2, 16, 16, 128, 128, 128, 64
    a = rnd(B, H, W, C, seed=1)
    s1, s2 = rnd(B, H, W, C1, seed=2), rnd(B, H, W, C2, seed=3)
    w = rnd(N, C, 3, 3, seed=4, scale=(9 * C) ** -0.5)
    ws = rnd(N, C1 + C2, 1, 1, seed=5, scale=(C1 + C2) ** -0.5)
    bias = rnd(B, N, seed=6, dtype=torch.float32)
    resid = rnd(B, H, W, N, seed=7)
    out = ops.conv3x3(a, pack_conv_w(w, [ws]), bias=bias, bias_bstride=N, skip1=s1, skip2=s2, resid=resid)
    ref = F.conv2d(a.float().permute(0, 3, 1, 2), w.float(), padding=1)
    ref = ref + F.conv2d(torch.cat([s1, s2], -1).float().permute(0, 3, 1, 2), ws.float())
    ref = ref + bias[:, :, None, None] + resid.float().permute(0, 3, 1, 2)
    assert_close(out, ref.permute(0, 2, 3, 1), what="conv resblock tail")


def build_attention_inputs(ops, q, k, v):
    """q [B,H,Nq,d], k/v [B,H,Nk,d] fp32 -> padded kernel layouts (kv stride padded to 8 per batch item)"""
    B, H, Nq, d = q.shape
    Nk = k.shape[2]
    Nkp = (Nk + 7) // 8 * 8
    dk, dv = ops.attention_pads(d)
    Q = torch.zeros(B * Nq, H * dk, dtype=torch.bfloat16, device=DEV)
    K = torch.zeros(B * Nkp, H * dk, dtype=torch.bfloat16, device=DEV)
    Vt = torch.zeros(H * dv, B * Nkp, dtype=torch.bfloat16, device=DEV)
    Q.view(B, Nq, H, dk)[..., :d] = q.permute(0, 2, 1, 3).to(torch.bfloat16)
    K.view(B, Nkp, H, dk)[:, :Nk, :, :d] = k.permute(0, 2, 1, 3).to(torch.bfloat16)
    Vt.view(H, dv, B, Nkp)[:, :d, :, :Nk] = v.permute(1, 3, 0, 2).to(torch.bfloat16)
    if Nkp != Nk:  # poison the pad keys: the kernel must mask them, not rely on zeros
        K.view(B, Nkp, H, dk)[:, Nk:] = 7.0
        Vt.view(H, dv, B, Nkp)[:, :, :, Nk:] = 1000.0
    return Q, K, Vt, Nkp


ATT_CASES = [
    # B, H, Nq, Nk, d, causal
    (1, 2, 128, 128, 40, False),
    (2, 8, 256, 256, 40, False),
    (1, 2, 4096, 4096, 40, False),
    (2, 8, 1024, 77, 80, False),
    (2, 8, 64, 64, 160, False),
    (2, 8, 256, 257, 160, False),
    (2, 8, 1024, 1028, 80, False),
    (2, 12, 77, 77, 64, True),
    (2, 16, 257, 257, 64, False),
    (3, 8, 4096, 77, 40, False),
    # longer key ranges, ragged tails and the d_head <= 64 instantiations (attention_kernel<DK 64, DVP 48 / 64>)
    (2, 8, 1024, 1024, 40, False),
    (2, 4, 512, 640, 64, False),       # d 64: all four K16 steps, DVP 64
    (1, 3, 256, 1000, 40, False),      # masked tail tile (1000 = 7 * 128 + 104)
    (2, 2, 768, 520, 48, False),       # d 48; kv stride 520, five tiles, last one 8 keys
    (8, 8, 4096, 4096, 40, False),     # the benchmark's own self-attention launch (B = 8, 64x64 latent)
    (2, 3, 512, 900, 56, False),       # d 56 in DVP 64: row sums through the ones row of V^T, masked tail
    (1, 2, 256, 512, 32, False),       # d 32 in DVP 48: two padding swizzle groups behind the data rows
    (1, 8, 1024, 1028, 40, False),     # four token-concatenated image contexts (4 x 257 keys, app.py mcg tab): 8 full tiles + 4 keys
    (2, 8, 256, 514, 80, False),       # two images at d_head 80 (attention_kernel<DK 128, DVP 80>, masked tail tile)
]


@pytest.mark.parametrize("B,H,Nq,Nk,d,causal", ATT_CASES)
def test_attention(B, H, Nq, Nk, d, causal):
    ops = _ops()
    q, k, v = (rnd(B, H, n, d, seed=s, dtype=torch.float32) for s, n in ((1, Nq), (2, Nk), (3, Nk)))
    q = q * 2.0  # make the softmax peaky enough to exercise the rescale path
    Q, K, Vt, Nkp = build_attention_inputs(ops, q, k, v)
    out = torch.empty(B * Nq, H * d, dtype=torch.bfloat16, device=DEV)
    ops.attention(Q, K, Vt, out, B, H, Nq, Nk, d, causal=causal, kv_bstride=Nkp)
    qb, kb, vb = (t.to(torch.bfloat16).float() for t in (q, k, v))
    sim = torch.einsum("bhid,bhjd->bhij", qb, kb) * d ** -0.5
    if causal:
        sim = sim + torch.full((Nq, Nk), float("-inf"), device=DEV).triu(1)
    ref = torch.einsum("bhij,bhjd->bhid", sim.softmax(-1), vb).permute(0, 2, 1, 3).reshape(B * Nq, H * d)
    assert_close(out, ref, what=f"attention B{B} H{H} {Nq}x{Nk} d{d}")


@pytest.mark.parametrize("B,HW,C1,C2,act,eps", [(2, 4096, 320, 0, 1, 1e-5), (2, 1024, 640, 320, 1, 1e-5),
                                              (3, 64, 1280, 1280, 1, 1e-5), (2, 256, 1280, 640, 0, 1e-6),
                                              (1, 65536, 128, 0, 1, 1e-6), (2, 4096, 512, 0, 0, 1e-6),
                                              # UNet batch (B = 8): few CTAs per image -> the generic two-read path at the
                                              # large layers, the register-resident path at the small ones
                                              (8, 4096, 320, 0, 1, 1e-5), (8, 1024, 640, 640, 1, 1e-5),
                                              (8, 256, 1280, 1280, 1, 1e-5), (8, 64, 1280, 0, 1, 1e-5),
                                              (8, 100, 320, 0, 0, 1e-6),
                                              # group-bundle kernel: cluster sizes 1..8, bundles that straddle the two concat
                                              # sources (C1 = 1280 | 640 at 60 channels per group), odd pixel counts
                                              (8, 4096, 320, 320, 1, 1e-5), (8, 1024, 1280, 640, 1, 1e-5), (8, 256, 1280, 640, 1, 1e-5),
                                              (8, 1024, 640, 320, 1, 1e-5), (8, 4096, 640, 320, 1, 1e-5), (8, 64, 1280, 1280, 1, 1e-5),
                                              (2, 577, 320, 0, 1, 1e-5), (4, 1024, 128, 0, 1, 1e-6), (4, 4096, 256, 0, 0, 1e-6),
                                              (3, 36, 640, 640, 1, 1e-5), (1, 16384, 512, 0, 1, 1e-6)])
def test_groupnorm(B, HW, C1, C2, act, eps):
    ops = _ops()
    x1 = rnd(B, HW, C1, seed=1) + 0.5
    x2 = rnd(B, HW, C2, seed=2, scale=2.0) if C2 else None
    C = C1 + C2
    g, b = rnd(C, seed=3, dtype=torch.float32), rnd(C, seed=4, dtype=torch.float32)
    out = ops.groupnorm(x1, g, b, eps, act=act, x2=x2)
    x = torch.cat([x1, x2], -1) if C2 else x1
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, g, b, eps)
    if act:
        ref = F.silu(ref)
    assert_close(out, ref.permute(0, 2, 1), tol=1.5e-2, what="groupnorm")
    out2 = ops.groupnorm(x1, g, b, eps, act=act, x2=x2)
    assert torch.equal(out, out2), "groupnorm must be run-to-run deterministic"


@pytest.mark.parametrize("rows,C", [(4096, 320), (1000, 640), (512, 1280), (154, 768), (514, 1024), (32768, 320), (4099, 320),
                                    (3, 320), (517, 64), (130, 128), (77, 256), (64, 2048), (100, 1000 // 8 * 8)])
def test_layernorm(rows, C):
    ops = _ops()
    x = rnd(rows, C, seed=1) * 3 + 1
    g, b = rnd(C, seed=3, dtype=torch.float32), rnd(C, seed=4, dtype=torch.float32)
    out = ops.layernorm(x, g, b, 1e-5)
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5)
    assert_close(out, ref, tol=1.5e-2, what="layernorm")


def test_upsample_im2col_permute_cast():
    ops = _ops()
    x = rnd(2, 8, 8, 64, seed=1)
    up = ops.upsample2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), ref)
    z = rnd(2, 4, 16, 16, seed=2, dtype=torch.float32)
    zh = ops.nchw_to_nhwc(z)
    assert torch.equal(zh, z.permute(0, 2, 3, 1).contiguous())
    back = ops.nhwc_to_nchw(zh, mul=0.5, add=0.5, clamp01=True)
    assert torch.equal(back, torch.clamp(z * 0.5 + 0.5, 0, 1))
    col = ops.im2col3x3_small(zh, kpad=64)
    unf = F.unfold(z, 3, padding=1)  # [B, C*9, L] with (c, ky, kx) order
    unf = unf.view(2, 4, 9, 256).permute(0, 3, 2, 1).reshape(2 * 256, 36)  # -> (tap, c)
    assert torch.equal(col[:, :36].float(), unf.to(torch.bfloat16).float())
    assert (col[:, 36:] == 0).all()
    assert torch.equal(ops.to_f32(ops.to_bf16(z)), z.to(torch.bfloat16).float())


def test_timestep_embedding_and_linear_small():
    ops = _ops()
    ts = torch.tensor([1, 21, 501, 981, 999, 0, 7, 333], dtype=torch.int64, device=DEV)
    emb = ops.timestep_embedding(ts, 320)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half).to(DEV)
    args = ts[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
    assert (emb - ref).abs().max().item() <= 2e-4   # fp32 sin/cos of arguments up to 1e3 (1 ulp of freq moves the argument by 1e-4)
    table = torch.tensor([981, 961, 941], dtype=torch.int64, device=DEV)
    idx = torch.tensor([1], dtype=torch.int32, device=DEV)
    emb2 = ops.timestep_embedding(table, 320, step_idx=idx, batch=4)
    assert torch.equal(emb2, ops.timestep_embedding(torch.full((4,), 961, dtype=torch.int64, device=DEV), 320))
    w = rnd(1280, 320, seed=5, scale=320 ** -0.5)
    b = rnd(1280, seed=6, dtype=torch.float32)
    h = ops.linear_small(emb, w, b, act_out=ops.ACT_SILU)
    refh = F.silu(emb @ w.float().t() + b)
    assert_close(h, refh, tol=1e-4, cos_min=0.99999, what="linear_small")
    w2 = rnd(5000, 1280, seed=7, scale=1280 ** -0.5)
    o = ops.linear_small(h, w2, None, act_in=ops.ACT_SILU)
    assert_close(o, F.silu(h) @ w2.float().t(), tol=1e-4, cos_min=0.99999, what="linear_small silu-in")


def test_softmax_rows():
    ops = _ops()
    x = rnd(300, 4096, seed=1, scale=4.0)
    out = ops.softmax_rows(x, scale=0.044)
    ref = (x.float() * 0.044).softmax(-1)
    assert_close(out, ref, tol=1e-2, what="softmax_rows")


def test_weight_repack_abi_matches_the_python_packers():
    """vdb_pack_conv_weight / vdb_pack_geglu / vdb_pad_heads (include/vdb200.h) produce exactly the layouts that
    lib/model_zoo's PackedModule._pack builds in Python (bit-identical bf16)."""
    ops = _ops()
    from lib.model_zoo.diffusion_utils import pack_conv3x3, pack_conv1x1
    from lib.model_zoo.attention import GEGLU, CrossAttention
    g = torch.Generator().manual_seed(5)
    w3 = torch.randn(96, 40, 3, 3, generator=g).to(DEV)
    w1 = torch.randn(96, 24, 1, 1, generator=g).to(DEV)
    ref = torch.cat([pack_conv3x3(w3), pack_conv1x1(w1)], dim=1)
    out = torch.empty_like(ref)
    ops.pack_conv_weight(w3, out=out, col0=0)
    ops.pack_conv_weight(w1, out=out, col0=9 * 40)
    assert torch.equal(out, ref)
    gl = GEGLU(64, 256).to(DEV)
    p = gl.packed()
    wo, bo = ops.pack_geglu(gl.proj.weight.detach().float().contiguous(), gl.proj.bias.detach().float().contiguous())
    assert torch.equal(wo, p["w"]) and torch.equal(bo, p["b"])
    ca = CrossAttention(320, context_dim=768, heads=8, dim_head=40).to(DEV)
    pk = ca.packed()
    assert torch.equal(ops.pad_heads(ca.to_q.weight.detach().float().contiguous(), 8, 40, pk["dk"]), pk["wq"])
    assert torch.equal(ops.pad_heads(ca.to_v.weight.detach().float().contiguous(), 8, 40, pk["dv"]), pk["wv"])
