"""Torch-tensor front end of the vdb200 C ABI (include/vdb200.h).

torch is used here for device memory, streams and allocation only; every arithmetic op on the hot
path is a kernel of libvdb200.so.  All functions enqueue on torch's current CUDA stream and are
CUDA-graph capturable (no host syncs, scratch comes from the caller or torch's caching allocator).
"""
import ctypes
import math

import torch

from ._lib import lib, check

ACT_NONE, ACT_SILU, ACT_GELU, ACT_QUICK_GELU, ACT_GEGLU = 0, 1, 2, 3, 4
BF16 = torch.bfloat16


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _need(t, dtype, name, rows_ok=False):
    if t is None:
        return
    if not t.is_cuda:
        raise ValueError(f"{name}: vdb200 kernels need CUDA tensors (no CPU fallback)")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    if rows_ok and t.dim() == 2 and t.stride(1) == 1:
        return  # row-strided 2-D view: the kernels take a leading dimension
    if not t.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")


_workspace = {}
WORKSPACE_BYTES = 160 << 20   # covers 16-way split-K of any MN grid that fits in half the SMs (74 tiles x 128 x 256 fp32)


def _scratch_key(device):
    """(device, stream) key of the split-K workspace / GroupNorm scratch.  The C ABI promises reuse of a scratch buffer on ONE
    stream only (the GroupNorm arrival counters and the split-K partials are not re-entrant), so every eager stream gets its
    own buffers: two threads sampling on two streams of one GPU no longer share counters.  Launches issued while a CUDA graph
    is being captured (torch captures on a side stream) use the buffers of the device's FIRST stream — the one the eager
    warm-up step ran on — so the addresses baked into the graph are the ones that were sized and zeroed before capture.
    Graphs captured from different streams therefore still share one scratch set and must not be replayed concurrently."""
    dev = device.index if device.index is not None else torch.cuda.current_device()
    sid = torch.cuda.current_stream(dev).cuda_stream
    owner = _scratch_owner.setdefault(dev, sid)
    if torch.cuda.is_current_stream_capturing():
        sid = owner
    return (dev, sid)


_scratch_owner = {}


def workspace(device):
    """Fixed-size fp32 split-K scratch per (device, stream). Never reallocated: its address is baked into captured CUDA graphs."""
    key = _scratch_key(device)
    w = _workspace.get(key)
    if w is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("split-K workspace must exist before CUDA-graph capture (run one eager step first)")
        w = torch.empty(WORKSPACE_BYTES // 4, dtype=torch.float32, device=device)
        _workspace[key] = w
    return w


# ------------------------------------------------------------------------------------------------
# optional per-family device timing (bench.py roofline leg): CUDA events on the launching stream
# ------------------------------------------------------------------------------------------------
_PROFILE = None


class _Span(object):
    __slots__ = ("name", "flops", "nbytes", "e0", "e1")

    def __init__(self, name, flops, nbytes):
        self.name, self.flops, self.nbytes = name, flops, nbytes

    def __enter__(self):
        if _PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _PROFILE is not None:
            self.e1.record()
            _PROFILE.append(self)
        return False


def profile_start():
    global _PROFILE
    _PROFILE = []


def profile_stop():
    """-> {family: {"ms": total, "launches": n, "flops": total, "bytes": total}}"""
    global _PROFILE
    spans, _PROFILE = _PROFILE, None
    torch.cuda.synchronize()
    out = {}
    for sp in spans or []:
        d = out.setdefault(sp.name, {"ms": 0.0, "launches": 0, "flops": 0.0, "bytes": 0.0})
        d["ms"] += sp.e0.elapsed_time(sp.e1)
        d["launches"] += 1
        d["flops"] += sp.flops
        d["bytes"] += sp.nbytes
    return out


# ------------------------------------------------------------------------------------------------
# optional recording of the tensor-core GEMM / conv launches (bench.py: replay of exactly these launches inside a CUDA
# graph, so the roofline leg can time the kernel without the host launch path).  Each record keeps its tensors alive.
# ------------------------------------------------------------------------------------------------
_RECORD = None


def record_start():
    global _RECORD
    _RECORD = []


def record_stop():
    """-> [(C function, arguments without the stream, tensors kept alive, algorithmic FLOPs)]"""
    global _RECORD
    rec, _RECORD = _RECORD, None
    return rec or []


def replay(records):
    """Re-issue recorded launches on the current stream (capturable)."""
    for fn, cargs, _keep, _flops in records:
        check(fn(*cargs, _stream()), "replay")


_gn_scratch_buf = {}


def _gn_scratch(device, nfloats):
    """Persistent zero-initialised GroupNorm scratch per (device, stream) (the kernels restore its counters to zero)."""
    key = _scratch_key(device)
    buf = _gn_scratch_buf.get(key)
    if buf is None or buf.numel() < nfloats:
        if buf is not None and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("GroupNorm scratch must be sized before CUDA-graph capture (run one eager step first)")
        buf = torch.zeros(max(int(nfloats), 1 << 20), dtype=torch.float32, device=device)
        _gn_scratch_buf[key] = buf
    return buf


def launch_count():
    return int(lib.vdb_launch_count())


def reset_launch_count():
    lib.vdb_reset_launch_count()


# ------------------------------------------------------------------------------------------------
def ddim_cfg_step(e_uncond, e_cond, x, coef, scale, x_prev=None, pred_x0=None, noise=None,
                  temperature=1.0, step_idx=None, x_prev_dup=None):
    """K4 (ddim.py:144-171). e_*/x/noise fp32 same shape; coef fp32 [.,4] device tensor."""
    for n, t in (("e_uncond", e_uncond), ("e_cond", e_cond), ("x", x), ("noise", noise), ("coef", coef)):
        _need(t, torch.float32, n)
    if x_prev is None:
        x_prev = torch.empty_like(x)
    if step_idx is not None:
        _need(step_idx, torch.int32, "step_idx")
    check(lib.vdb_ddim_cfg_step(_ptr(e_uncond), _ptr(e_cond), _ptr(x), _ptr(noise), _ptr(coef), _ptr(step_idx),
                                float(scale), float(temperature), _ptr(x_prev), _ptr(x_prev_dup), _ptr(pred_x0), x.numel(),
                                _stream()),
          "ddim_cfg_step")
    return x_prev, pred_x0


def dpmpp_cfg_step(e_uncond, e_cond, x, coef, step_idx, scale, hist, x_next=None, x_next_dup=None, pred_x0=None, seed=None,
                   noise=None):
    """CFG mix + one multistep DPM-Solver++ update (lib/model_zoo/dpm_solver.py).  e_*/x fp32 of n elements; coef fp32 [., 8]
    device table, row step_idx[0] (int32 device tensor); hist fp32 ring of 3 n elements.  With seed (int64 device word keying the
    Philox draws) or noise (fp32 of n elements, used instead of the draws) the step is the SDE form, vdb_dpmpp_sde_cfg_step: row
    column 6 scales the noise term.  With neither it is vdb_dpmpp_cfg_step."""
    for name, t in (("e_uncond", e_uncond), ("e_cond", e_cond), ("x", x), ("coef", coef), ("hist", hist),
                    ("x_next_dup", x_next_dup), ("pred_x0", pred_x0), ("noise", noise)):
        _need(t, torch.float32, name)
    _need(step_idx, torch.int32, "step_idx")
    _need(seed, torch.int64, "seed")
    if coef.dim() != 2 or coef.shape[1] != 8:
        raise ValueError(f"coef: expected [rows, 8], got {tuple(coef.shape)}")
    n = x.numel()
    if hist.numel() != 3 * n:
        raise ValueError(f"hist: expected 3 x {n} elements, got {hist.numel()}")
    if noise is not None and noise.numel() != n:
        raise ValueError(f"noise: expected {n} elements, got {noise.numel()}")
    if x_next is None:
        x_next = torch.empty_like(x)
    if seed is None and noise is None:
        check(lib.vdb_dpmpp_cfg_step(_ptr(e_uncond), _ptr(e_cond), _ptr(x), _ptr(coef), _ptr(step_idx), float(scale), _ptr(hist),
                                     _ptr(x_next), _ptr(x_next_dup), _ptr(pred_x0), n, _stream()),
              "dpmpp_cfg_step")
    else:
        check(lib.vdb_dpmpp_sde_cfg_step(_ptr(e_uncond), _ptr(e_cond), _ptr(x), _ptr(coef), _ptr(step_idx), float(scale),
                                         _ptr(hist), _ptr(x_next), _ptr(x_next_dup), _ptr(pred_x0), n, _ptr(seed), _ptr(noise),
                                         _stream()),
              "dpmpp_sde_cfg_step")
    return x_next, pred_x0


def inpaint_blend(x, x0, mask, table, step_idx, seed=None, noise=None, x_dup=None):
    """Inpainting blend after a sampler step (lib/model_zoo/inpaint.py), in place on x.  x / x0 / noise / x_dup fp32 NHWC
    [bs, H, W, C]; mask fp32 of H*W (broadcast over the batch) or bs*H*W elements; table fp32 [., 2] device rows, row
    step_idx[0] (int32 device tensor); seed int64 device word keying the Philox draws, unused when noise is given."""
    for name, t in (("x", x), ("x0", x0), ("mask", mask), ("table", table), ("noise", noise), ("x_dup", x_dup)):
        _need(t, torch.float32, name)
    _need(step_idx, torch.int32, "step_idx")
    _need(seed, torch.int64, "seed")
    bs, C = x.shape[0], x.shape[-1]
    hw = x.numel() // (bs * C)
    for name, t in (("x0", x0), ("noise", noise), ("x_dup", x_dup)):
        if t is not None and t.shape != x.shape:
            raise ValueError(f"{name}: expected {tuple(x.shape)}, got {tuple(t.shape)}")
    if mask.numel() not in (hw, bs * hw):
        raise ValueError(f"mask: expected {hw} or {bs * hw} elements, got {mask.numel()}")
    if table.dim() != 2 or table.shape[1] != 2:
        raise ValueError(f"table: expected [rows, 2], got {tuple(table.shape)}")
    check(lib.vdb_inpaint_blend_f32(_ptr(x), _ptr(x_dup), _ptr(x0), _ptr(mask), int(mask.numel() != hw), _ptr(table),
                                    _ptr(step_idx), _ptr(seed), _ptr(noise), bs, hw, C, _stream()),
          "inpaint_blend")
    return x


def inpaint_noise(seed, step_idx, n, out=None):
    """The inpainting blend's Philox draws at step step_idx[0] for the first n elements of a latent -> fp32 [n]."""
    _need(seed, torch.int64, "seed")
    _need(step_idx, torch.int32, "step_idx")
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=seed.device)
    _need(out, torch.float32, "out")
    check(lib.vdb_inpaint_noise_f32(_ptr(seed), _ptr(step_idx), int(n), _ptr(out), _stream()), "inpaint_noise")
    return out


def mask_to_latent(mask, out=None):
    """Pixel mask fp32 [n, 1, 8H, 8W] -> latent mask [n, 1, H, W], the max over each 8x8 cell."""
    _need(mask, torch.float32, "mask")
    if mask.dim() != 4 or mask.shape[1] != 1 or mask.shape[2] % 8 or mask.shape[3] % 8:
        raise ValueError(f"mask: expected [n, 1, 8H, 8W], got {tuple(mask.shape)}")
    n, _, H8, W8 = mask.shape
    if out is None:
        out = torch.empty((n, 1, H8 // 8, W8 // 8), dtype=torch.float32, device=mask.device)
    check(lib.vdb_mask_to_latent(_ptr(mask), n, H8, W8, _ptr(out), _stream()), "mask_to_latent")
    return out


def composite(decoded, image, mask, out=None):
    """out = m*decoded + (1 - m)*image per pixel: decoded / image fp32 NCHW [n, C, H, W], mask fp32 [n or 1, 1, H, W]."""
    for name, t in (("decoded", decoded), ("image", image), ("mask", mask)):
        _need(t, torch.float32, name)
    if decoded.dim() != 4 or image.shape != decoded.shape:
        raise ValueError(f"image: expected {tuple(decoded.shape)}, got {tuple(image.shape)}")
    n, C, H, W = decoded.shape
    if mask.dim() != 4 or mask.shape[0] not in (1, n) or tuple(mask.shape[1:]) != (1, H, W):
        raise ValueError(f"mask: expected [{n} or 1, 1, {H}, {W}], got {tuple(mask.shape)}")
    if out is None:
        out = torch.empty_like(decoded)
    check(lib.vdb_composite_f32(_ptr(decoded), _ptr(image), _ptr(mask), int(mask.shape[0] != 1), n, C, H * W, _ptr(out),
                                _stream()),
          "composite")
    return out


def latent_store_slot(x, ring, step_idx, offset):
    """ring[step_idx[0] + offset] = x (lib/model_zoo/edit.py): x fp32 of n elements, ring fp32 [slots, ...] of slots * n."""
    _need(x, torch.float32, "x")
    _need(ring, torch.float32, "ring")
    _need(step_idx, torch.int32, "step_idx")
    n = x.numel()
    if ring.dim() < 1 or ring.numel() != ring.shape[0] * n:
        raise ValueError(f"ring: expected [slots, {tuple(x.shape)}], got {tuple(ring.shape)}")
    check(lib.vdb_latent_store_slot_f32(_ptr(x), _ptr(ring), ring.shape[0], _ptr(step_idx), int(offset), n, _stream()),
          "latent_store_slot")
    return ring


def inversion_blend(x, ring, mask, step_idx, x_dup=None):
    """x = m x + (1 - m) ring[step_idx[0]] after a step of a walk from an inversion (lib/model_zoo/edit.py), in place on x.  x /
    x_dup fp32 NHWC [bs, H, W, C]; ring fp32 [slots, bs, H, W, C]; mask fp32 of H*W (broadcast over the batch) or bs*H*W."""
    for name, t in (("x", x), ("ring", ring), ("mask", mask), ("x_dup", x_dup)):
        _need(t, torch.float32, name)
    _need(step_idx, torch.int32, "step_idx")
    bs, C = x.shape[0], x.shape[-1]
    hw = x.numel() // (bs * C)
    if x_dup is not None and x_dup.shape != x.shape:
        raise ValueError(f"x_dup: expected {tuple(x.shape)}, got {tuple(x_dup.shape)}")
    if ring.dim() != x.dim() + 1 or tuple(ring.shape[1:]) != tuple(x.shape):
        raise ValueError(f"ring: expected [slots, {', '.join(map(str, x.shape))}], got {tuple(ring.shape)}")
    if mask.numel() not in (hw, bs * hw):
        raise ValueError(f"mask: expected {hw} or {bs * hw} elements, got {mask.numel()}")
    check(lib.vdb_inversion_blend_f32(_ptr(x), _ptr(x_dup), _ptr(ring), ring.shape[0], _ptr(mask), int(mask.numel() != hw),
                                      _ptr(step_idx), bs, hw, C, _stream()),
          "inversion_blend")
    return x


def diffedit_mask(e_src_u, e_src_c, s_src, e_tgt_u, e_tgt_c, s_tgt, D, ratio, out=None):
    """DiffEdit's {0, 1} mask (lib/model_zoo/edit.py) -> fp32 [bs, H, W].  e_* fp32 NHWC [D*bs, H, W, C], draw d of image b at row
    d*bs + b; an e_*_u is None when that side has no CFG."""
    for name, t in (("e_src_u", e_src_u), ("e_src_c", e_src_c), ("e_tgt_u", e_tgt_u), ("e_tgt_c", e_tgt_c)):
        _need(t, torch.float32, name)
        if t is not None and t.shape != e_src_c.shape:
            raise ValueError(f"{name}: expected {tuple(e_src_c.shape)}, got {tuple(t.shape)}")
    D = int(D)
    if D < 1:
        raise ValueError(f"D must be >= 1, got {D}")
    if e_src_c.dim() != 4 or e_src_c.shape[0] % D:
        raise ValueError(f"eps: expected [D*bs, H, W, C] with D = {D}, got {tuple(e_src_c.shape)}")
    R, H, W, C = e_src_c.shape
    bs = R // D
    if out is None:
        out = torch.empty(bs, H, W, dtype=torch.float32, device=e_src_c.device)
    _need(out, torch.float32, "out")
    if out.numel() != bs * H * W:
        raise ValueError(f"out: expected {bs * H * W} elements ([{bs}, {H}, {W}]), got {tuple(out.shape)}")
    check(lib.vdb_diffedit_mask_f32(_ptr(e_src_u), _ptr(e_src_c), float(s_src), _ptr(e_tgt_u), _ptr(e_tgt_c), float(s_tgt), int(D),
                                    bs, H * W, C, float(ratio), _ptr(out), _stream()),
          "diffedit_mask")
    return out


def _same_shape(ref, t, name):
    if t is not None and t.shape != ref.shape:
        raise ValueError(f"{name}: expected {tuple(ref.shape)}, got {tuple(t.shape)}")


def axpby(x, z, a, b, out=None):
    _need(x, torch.float32, "x"); _need(z, torch.float32, "z"); _need(out, torch.float32, "out")
    _same_shape(x, z, "z")
    _same_shape(x, out, "out")
    if out is None:
        out = torch.empty_like(x)
    check(lib.vdb_axpby_f32(_ptr(x), _ptr(z), float(a), float(b), _ptr(out), x.numel(), _stream()), "axpby")
    return out


def lincomb4(xs, cs, out=None):
    """sum_i cs[i] * xs[i] for 1..4 fp32 tensors of one shape."""
    if not 1 <= len(xs) <= 4 or len(xs) != len(cs):
        raise ValueError(f"lincomb4: need 1 to 4 tensors and as many coefficients, got {len(xs)} and {len(cs)}")
    for i, t in enumerate(xs):
        _need(t, torch.float32, f"xs[{i}]")
        _same_shape(xs[0], t, f"xs[{i}]")
    _need(out, torch.float32, "out")
    _same_shape(xs[0], out, "out")
    if out is None:
        out = torch.empty_like(xs[0])
    ptrs = [_ptr(t) for t in xs] + [0] * (4 - len(xs))
    coef = [float(c) for c in cs] + [0.0] * (4 - len(cs))
    check(lib.vdb_lincomb4_f32(ptrs[0], ptrs[1], ptrs[2], ptrs[3], coef[0], coef[1], coef[2], coef[3], _ptr(out),
                               xs[0].numel(), _stream()), "lincomb4")
    return out


def add_int(t, delta):
    _need(t, torch.int32, "counter")
    check(lib.vdb_add_int(_ptr(t), int(delta), _stream()), "add_int")


def gemm(a, w, bias=None, resid=None, out=None, act=ACT_NONE, a2=None, out_dtype=BF16, alpha=1.0,
         bias_bstride=0, rows_per_batch=1, bn=0, ksplit=0):
    """out[M,N'] = act(alpha*[a|a2] @ w^T + bias) + resid ; a [M,K] bf16, w [N,K(+K2)] bf16."""
    _need(a, BF16, "a", True); _need(w, BF16, "w", True); _need(a2, BF16, "a2", True); _need(bias, torch.float32, "bias")
    _need(resid, BF16, "resid", True)
    M, K = a.shape
    N = w.shape[0]
    K2 = a2.shape[1] if a2 is not None else 0
    assert w.shape[1] == K + K2, (w.shape, K, K2)
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=out_dtype, device=a.device)
    _need(out, out_dtype, "out", True)
    ws, ws_bytes = None, 0
    if ksplit != 1 and M <= 8192:   # split-K only ever triggers for small MN grids
        ws, ws_bytes = workspace(a.device), WORKSPACE_BYTES
    cargs = (_ptr(a), M, K, a.stride(0), _ptr(a2), K2, a2.stride(0) if a2 is not None else 0,
             _ptr(w), N, w.stride(0), _ptr(bias), int(bias_bstride), int(rows_per_batch),
             _ptr(resid), resid.stride(0) if resid is not None else 0, _ptr(out), out.stride(0),
             1 if out_dtype == torch.float32 else 0, int(act), float(alpha), int(bn), int(ksplit),
             _ptr(ws), ws_bytes)
    with _Span("gemm", 2.0 * M * N * (K + K2), 2.0 * (M * (K + K2) + N * (K + K2) + M * n_out)):
        check(lib.vdb_gemm_bf16(*cargs, _stream()), "gemm_bf16")
    if _RECORD is not None:
        _RECORD.append((lib.vdb_gemm_bf16, cargs, (a, a2, w, bias, resid, out, ws), 2.0 * M * N * (K + K2)))
    return out


IGEMM_PLAN_FIELDS = ("bn", "stages", "mode", "ksplit", "grid", "tiles_m", "tiles_n", "bm", "n_fast")   # (bm, n_fast: their own accessors)
BM256 = 0x1000      # VDB_IGEMM_BM256: bn=160 | BM256 forces the 256-row tile of gemm / gemm_ln / conv3x3


def igemm_last_plan():
    """The tiling of the last gemm / gemm_ln / conv3x3 launch on this thread (vdb_igemm_last_plan): which kernel instantiation
    (BM, BN, STAGES, epilogue MODE) ran, with its split-K factor, grid and tile counts, and whether it walked its tiles N-fast."""
    buf = (ctypes.c_int * (len(IGEMM_PLAN_FIELDS) - 2))()
    n = lib.vdb_igemm_last_plan(buf, len(buf))
    assert n == len(buf), n
    return dict(zip(IGEMM_PLAN_FIELDS, list(buf) + [lib.vdb_igemm_last_bm(), lib.vdb_igemm_last_n_fast()]))


class LnFold(object):
    """What a GEMM needs to consume a LayerNorm it never sees (vdb_gemm_ln_bf16): the producer's partial sums `stats`
    [>= parts, rows, 2] fp32 (`parts` of them valid), the LayerNorm's width and epsilon; the weights' column sums ride with the
    packed weights."""

    def __init__(self, stats, parts, dim, eps):
        self.stats, self.parts, self.dim, self.eps = stats, int(parts), int(dim), float(eps)


def ln_stats_buffer(rows, width, device):
    """statistics table a producer GEMM with N = width columns fills for its `rows` output rows (worst case: 64-column tiles)"""
    assert width % 32 == 0
    return torch.empty((2 * ((width + 63) // 64), rows, 2), dtype=torch.float32, device=device)


def gemm_ln(a, w, bias=None, resid=None, out=None, act=ACT_NONE, ln=None, colsum=None, on_cols=False, rowbias=None,
            stats_out=None, bn=0):
    """vdb_gemm_ln_bf16: consumer (ln = LnFold, colsum) or producer (stats_out; returns (out, parts)) of folded-LayerNorm
    statistics."""
    _need(a, BF16, "a", True); _need(w, BF16, "w", True); _need(bias, torch.float32, "bias"); _need(resid, BF16, "resid", True)
    _need(colsum, torch.float32, "colsum"); _need(rowbias, torch.float32, "rowbias"); _need(stats_out, torch.float32, "stats_out")
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K, (w.shape, K)
    n_out = N // 2 if act == ACT_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=BF16, device=a.device)
    _need(out, BF16, "out", True)
    st = None
    if ln is not None:
        st = ln.stats
        _need(st, torch.float32, "ln.stats")
        assert st.dim() == 3 and st.shape[0] >= ln.parts and st.shape[2] == 2, (tuple(st.shape), ln.parts)
    parts = ctypes.c_int(0)
    if stats_out is not None:
        assert stats_out.dim() == 3 and stats_out.shape[0] >= 2 * ((N + 63) // 64) and stats_out.shape[1] == M and stats_out.shape[2] == 2, \
            (tuple(stats_out.shape), N, M)
    cargs = (_ptr(a), M, K, a.stride(0), _ptr(w), N, w.stride(0), _ptr(bias), _ptr(resid),
             resid.stride(0) if resid is not None else 0, _ptr(out), out.stride(0), int(act),
             _ptr(st), st.shape[1] if st is not None else 0, ln.parts if ln is not None else 0, ln.dim if ln is not None else 0,
             ln.eps if ln is not None else 0.0, _ptr(colsum), 1 if on_cols else 0, _ptr(rowbias), _ptr(stats_out),
             ctypes.addressof(parts) if stats_out is not None else None, int(bn))
    with _Span("gemm", 2.0 * M * N * K, 2.0 * (M * K + N * K + M * n_out)):
        check(lib.vdb_gemm_ln_bf16(*cargs, _stream()), "gemm_ln_bf16")
    if _RECORD is not None:
        _RECORD.append((lib.vdb_gemm_ln_bf16, cargs, (a, w, bias, resid, out, st, colsum, rowbias, stats_out, parts), 2.0 * M * N * K))
    return (out, parts.value) if stats_out is not None else out


def conv3x3(x, w, bias=None, resid=None, out=None, mode=0, skip1=None, skip2=None, act=ACT_NONE,
            out_dtype=BF16, bias_bstride=0, bn=0, ksplit=0):
    """3x3 conv on NHWC bf16 x [B,H,W,C]; w [N, 9*C + Cs1 + Cs2] packed (ky,kx,c | skip)."""
    _need(x, BF16, "x"); _need(w, BF16, "w"); _need(bias, torch.float32, "bias")
    _need(resid, BF16, "resid"); _need(skip1, BF16, "skip1"); _need(skip2, BF16, "skip2")
    B, H, W, Cc = x.shape
    N = w.shape[0]
    Ho, Wo = (H // 2, W // 2) if mode in (1, 2) else (H, W)
    cs1 = skip1.shape[-1] if skip1 is not None else 0
    cs2 = skip2.shape[-1] if skip2 is not None else 0
    ntaps = 4 if mode >= 3 else 9          # modes 3..6 (7..10: stored interleaved into `out` [B,2H,2W,N]): folded nearest-2x upsample
    assert w.shape[1] == ntaps * Cc + cs1 + cs2, (w.shape, Cc, cs1, cs2, mode)
    if out is None:
        out = torch.empty((B, Ho, Wo, N), dtype=out_dtype, device=x.device)
    M = B * Ho * Wo
    ws, ws_bytes = None, 0
    if ksplit != 1 and M <= 8192:
        ws, ws_bytes = workspace(x.device), WORKSPACE_BYTES
    ktot = ntaps * Cc + cs1 + cs2
    cargs = (_ptr(x), B, H, W, Cc, int(mode), _ptr(w), N, w.stride(0), _ptr(skip1), cs1,
             _ptr(skip2), cs2, _ptr(bias), int(bias_bstride), _ptr(resid),
             resid.shape[-1] if resid is not None else 0, _ptr(out), out.shape[-1],
             1 if out_dtype == torch.float32 else 0, int(act), int(bn), int(ksplit), _ptr(ws), ws_bytes)
    with _Span("conv3x3", 2.0 * M * N * ktot, 2.0 * (B * H * W * Cc + M * (cs1 + cs2) + N * ktot + M * N)):
        check(lib.vdb_conv3x3_bf16(*cargs, _stream()), "conv3x3_bf16")
    if _RECORD is not None:
        _RECORD.append((lib.vdb_conv3x3_bf16, cargs, (x, w, skip1, skip2, bias, resid, out, ws), 2.0 * M * N * ktot))
    return out


def attention_pads(d_head):
    dk, dv = lib.vdb_attention_dk_pad(d_head), lib.vdb_attention_dv_pad(d_head)
    if dk < 0 or dv < 0:
        raise ValueError(f"d_head {d_head} unsupported by the attention kernel")
    return dk, dv


def attention(q, k, vt, out, B, H, Nq, Nk, d_head, scale=None, q_col0=0, k_col0=0, causal=False,
              q_bstride=0, kv_bstride=0, kv_len=None, items=None, step_idx=None, Bq=None, Bkv=None, accumulate=False):
    """Flash attention (vdb_attention_bf16). q [B*q_bstride, ldq], k [B*kv_bstride, ldk], vt [H*DVP, B*kv_bstride],
    out [B*q_bstride, H*d_head].  kv_bstride (default Nk) must be a multiple of 8: pad ragged contexts per batch item.
    kv_len (int32 device [B], d_head 64, not causal): item b attends to its first kv_len[b] keys only.
    items (int32 device [rows, 3, B]) with step_idx (int32 device [1]): output item b reads Q / K / V^T from items
    items[r, 0..2, b], r = step_idx[0], entries in [0, Bq) / [0, Bkv) (both default B), a negative V item skips b
    (lib/model_zoo/prompt_edit.py); accumulate: out += the attention (bf16)."""
    _need(q, BF16, "q", True); _need(k, BF16, "k", True); _need(vt, BF16, "vt", True); _need(out, BF16, "out", True)
    _need(kv_len, torch.int32, "kv_len"); _need(items, torch.int32, "items"); _need(step_idx, torch.int32, "step_idx")
    if items is not None:
        if items.dim() != 3 or items.shape[1] != 3 or items.shape[2] != B:
            raise ValueError(f"items: expected [rows, 3, {B}], got {tuple(items.shape)}")
        Bq = B if Bq is None else Bq
        Bkv = B if Bkv is None else Bkv
    if scale is None:
        scale = d_head ** -0.5
    with _Span("attention", 4.0 * B * H * Nq * Nk * d_head, 2.0 * B * H * d_head * (2 * Nq + 2 * Nk)):
        check(lib.vdb_attention_bf16(_ptr(q), q.stride(0), int(q_col0), _ptr(k), k.stride(0), int(k_col0), _ptr(vt), vt.stride(0),
                                     _ptr(out), out.stride(0), B, H, Nq, Nk, int(q_bstride), int(kv_bstride), d_head, float(scale),
                                     1 if causal else 0, _ptr(kv_len), int(Bq or 0), int(Bkv or 0), _ptr(items), _ptr(step_idx),
                                     1 if accumulate else 0, _stream()), "attention_bf16")
    return out


def xattn_word_map(q, k, w, out, row0, H, N, L, d_head, kv_bstride=0, scale=None):
    """Prompt-to-Prompt's word maps (vdb_xattn_word_map_f32): out[r, p] += sum_h sum_j w[r, j] softmax(scale q k^T)[h, p, j] for
    the n = w.shape[0] items row0 .. row0 + n - 1 of a cross-attention call's q [B*N, >= H*dk] and k [Bkv*kv_bstride, >= H*dk]."""
    _need(q, BF16, "q", True); _need(k, BF16, "k", True); _need(w, torch.float32, "w"); _need(out, torch.float32, "out")
    n = w.shape[0]
    if w.dim() != 2 or w.shape[1] != L:
        raise ValueError(f"w: expected [n, {L}], got {tuple(w.shape)}")
    if out.numel() != n * N:
        raise ValueError(f"out: expected {n * N} elements ([{n}, {N}]), got {tuple(out.shape)}")
    if scale is None:
        scale = d_head ** -0.5
    check(lib.vdb_xattn_word_map_f32(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(w), _ptr(out), n, int(row0), H, N, L,
                                     int(kv_bstride), d_head, float(scale), _stream()), "xattn_word_map")
    return out


def sattn_key_mass(q, k, mass, row0, H, N, d_head, w=1.0, q_col0=0, k_col0=0, kv_bstride=0, scale=None):
    """Self-attention guidance's key mass (vdb_sattn_key_mass_f32): mass[r, j] += w sum_h sum_p softmax(scale q k^T)[h, p, j] for
    the n = mass.shape[0] items row0 .. row0 + n - 1 of a self-attention call's q [B*N, >= q_col0 + H*dk] and k
    [B*kv_bstride, >= k_col0 + H*dk] (the fused q | k buffer passes the same tensor twice)."""
    _need(q, BF16, "q", True); _need(k, BF16, "k", True); _need(mass, torch.float32, "mass")
    if mass.dim() != 2 or mass.shape[1] != N:
        raise ValueError(f"mass: expected [n, {N}], got {tuple(mass.shape)}")
    n = mass.shape[0]
    if scale is None:
        scale = d_head ** -0.5
    stats = torch.empty(n * H * N * 2, dtype=torch.float32, device=mass.device)
    check(lib.vdb_sattn_key_mass_f32(_ptr(q), q.stride(0), int(q_col0), _ptr(k), k.stride(0), int(k_col0), _ptr(stats), float(w),
                                     _ptr(mass), n, int(row0), H, N, int(kv_bstride), d_head, float(scale), _stream()),
          "sattn_key_mass")
    return mass


def sag_degrade(x, e, mass, table, step_idx, hm, wm, out=None):
    """Self-attention guidance's degraded latent (vdb_sag_degrade_f32): x, e fp32 NHWC [bs, H, W, C]; mass fp32 [bs, hm*wm]; table
    fp32 [rows, 2] device rows {sqrt(a_t), sqrt(1 - a_t)}, row step_idx[0] (int32 device tensor) -> out [bs, H, W, C]."""
    for name, t in (("x", x), ("e", e), ("mass", mass), ("table", table), ("out", out)):
        _need(t, torch.float32, name)
    _need(step_idx, torch.int32, "step_idx")
    bs, H, W, C = x.shape
    if e.shape != x.shape:
        raise ValueError(f"e: expected {tuple(x.shape)}, got {tuple(e.shape)}")
    if mass.numel() != bs * hm * wm:
        raise ValueError(f"mass: expected [{bs}, {hm * wm}], got {tuple(mass.shape)}")
    if table.dim() != 2 or table.shape[1] != 2:
        raise ValueError(f"table: expected [rows, 2], got {tuple(table.shape)}")
    if out is None:
        out = torch.empty_like(x)
    elif out.shape != x.shape:
        raise ValueError(f"out: expected {tuple(x.shape)}, got {tuple(out.shape)}")
    check(lib.vdb_sag_degrade_f32(_ptr(x), _ptr(e), _ptr(mass), _ptr(table), _ptr(step_idx), bs, H, W, C, int(hm), int(wm),
                                  _ptr(out), _stream()), "sag_degrade")
    return out


def sag_guide(e_u, e_c, e_deg, s):
    """Self-attention guidance (vdb_sag_guide_f32), in place: d = s (e_src - e_deg), e_src = e_u when given (CFG) else e_c, is added
    to e_c and e_u.  All fp32 of one shape."""
    for name, t in (("e_u", e_u), ("e_c", e_c), ("e_deg", e_deg)):
        _need(t, torch.float32, name)
    for name, t in (("e_u", e_u), ("e_deg", e_deg)):
        if t is not None and t.shape != e_c.shape:
            raise ValueError(f"{name}: expected {tuple(e_c.shape)}, got {tuple(t.shape)}")
    check(lib.vdb_sag_guide_f32(_ptr(e_u), _ptr(e_c), _ptr(e_deg), float(s), e_c.numel(), _stream()), "sag_guide")


def local_blend(x, wmap, flags, step_idx, h, w, threshold, x_dup=None):
    """Prompt-to-Prompt's local blend after a step (vdb_local_blend_f32), in place on x fp32 NHWC [n, H, W, C] (row 0 the
    source): wmap fp32 [n, h*w] word maps, flags int32 device table read at step_idx[0]."""
    for name, t in (("x", x), ("wmap", wmap), ("x_dup", x_dup)):
        _need(t, torch.float32, name)
    _need(flags, torch.int32, "flags"); _need(step_idx, torch.int32, "step_idx")
    n, H, W, C = x.shape
    if x_dup is not None and x_dup.shape != x.shape:
        raise ValueError(f"x_dup: expected {tuple(x.shape)}, got {tuple(x_dup.shape)}")
    if wmap.numel() != n * h * w:
        raise ValueError(f"wmap: expected {n * h * w} elements ([{n}, {h}, {w}]), got {tuple(wmap.shape)}")
    check(lib.vdb_local_blend_f32(_ptr(x), _ptr(x_dup), _ptr(wmap), _ptr(flags), _ptr(step_idx), n, H, W, C, int(h), int(w),
                                  float(threshold), _stream()), "local_blend")
    return x


def _region_masks(masks, R, bs, H, W):
    if masks is not None and masks.numel() != R * bs * H * W:
        raise ValueError(f"masks: expected [{R}, {bs}, {H}, {W}], got {tuple(masks.shape)}")


def region_gather(x, oy, ox, h, w, first, k, R, u_blocks, out=None, masks=None, rows=None, step_idx=None, seed=None, bg=None,
                  noise=None):
    """Windows [first, first + k) of the canvas x fp32 NHWC [bs, H, W, C] -> the chunk batch out [(u_blocks + R + 1)*k*bs, h, w, C]
    of a region walk (lib/model_zoo/regions.py; R = 0 is a panorama's): u_blocks (0, 1 or R + 1) u blocks, then the R + 1 c blocks
    (row j*bs + b of a block: window first + j of image b).  oy / ox: int32 device origin tables.  Exact copies unless rows (fp32
    [., 4] {on, a, b, 0} device rows, row step_idx[0]) is on: then region r >= 1 reads m x + (1 - m) (a bg + b z) with masks fp32
    [R, bs, H, W], bg fp32 [nb, C] picked by the Philox stream keyed by seed (int64 device word), and z = noise (fp32 like x) when
    given, else that stream's normals."""
    for name, t in (("x", x), ("out", out), ("masks", masks), ("rows", rows), ("bg", bg), ("noise", noise)):
        _need(t, torch.float32, name)
    _need(oy, torch.int32, "oy"); _need(ox, torch.int32, "ox"); _need(step_idx, torch.int32, "step_idx")
    _need(seed, torch.int64, "seed")
    bs, H, W, C = x.shape
    shape = ((u_blocks + R + 1) * k * bs, h, w, C)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    if tuple(out.shape) != shape:
        raise ValueError(f"out: expected {shape}, got {tuple(out.shape)}")
    _region_masks(masks, R, bs, H, W)
    if noise is not None and noise.shape != x.shape:
        raise ValueError(f"noise: expected {tuple(x.shape)}, got {tuple(noise.shape)}")
    if bg is not None and (bg.dim() != 2 or bg.shape[1] != C):
        raise ValueError(f"bg: expected [nb, {C}], got {tuple(bg.shape)}")
    if rows is not None and (rows.dim() != 2 or rows.shape[1] != 4):
        raise ValueError(f"rows: expected [., 4], got {tuple(rows.shape)}")
    check(lib.vdb_region_gather_f32(_ptr(x), bs, H, W, C, _ptr(oy), _ptr(ox), oy.numel(), ox.numel(), int(h), int(w), int(first),
                                    int(k), int(R), int(u_blocks), _ptr(masks), _ptr(rows), _ptr(step_idx), _ptr(seed), _ptr(bg),
                                    0 if bg is None else bg.shape[0], _ptr(noise), _ptr(out), _stream()), "region_gather")
    return out


def region_noise(seed, step_idx, n, R, bs, nb):
    """The region gather's draws at step step_idx[0] -> (z fp32 [n] for the first n canvas elements, picks int32 [R, bs]: the
    background row of region r + 1, image b)."""
    _need(seed, torch.int64, "seed")
    _need(step_idx, torch.int32, "step_idx")
    z = torch.empty(n, dtype=torch.float32, device=seed.device)
    picks = torch.empty(R, bs, dtype=torch.int32, device=seed.device)
    check(lib.vdb_region_noise_f32(_ptr(seed), _ptr(step_idx), int(n), int(R), int(bs), int(nb), _ptr(z), _ptr(picks), _stream()),
          "region_noise")
    return z, picks


def region_merge(eps, oy, ox, cover_y, cover_x, first, k, R, masks, out, halves=1):
    """The mask-weighted merge of windows [first, first + k) of eps fp32 [halves*(R+1)*k*bs, h, w, C] (block s*(R+1) + r) into the
    canvas out [halves*bs, H, W, C] (lib/model_zoo/regions.py): the running fp32 sum over each element's covering windows in
    ascending window index, divided at the element's last one.  masks fp32 [R, bs, H, W], None when R = 0: then the merge is the
    plain window average of a panorama.  oy / ox / cover_y [H, 2] / cover_x [W, 4]: int32 device tables.  halves = 2 under CFG:
    eps is [u blocks; c blocks] and out [e_u; e_c]."""
    for name, t in (("eps", eps), ("out", out), ("masks", masks)):
        _need(t, torch.float32, name)
    for name, t in (("oy", oy), ("ox", ox), ("cover_y", cover_y), ("cover_x", cover_x)):
        _need(t, torch.int32, name)
    n, H, W, C = out.shape
    if halves not in (1, 2) or n % halves:
        raise ValueError(f"halves must be 1 or 2 and divide the {n} rows of out, got {halves}")
    bs = n // halves
    if eps.dim() != 4 or eps.shape[0] != (R + 1) * k * n or eps.shape[3] != C:
        raise ValueError(f"eps: expected [{(R + 1) * k * n}, h, w, {C}] for out {tuple(out.shape)}, got {tuple(eps.shape)}")
    _, h, w, _ = eps.shape
    _region_masks(masks, R, bs, H, W)
    if cover_y.numel() != 2 * H or cover_x.numel() != 4 * W:
        raise ValueError(f"cover tables: expected {2 * H} and {4 * W} entries, got {cover_y.numel()} and {cover_x.numel()}")
    check(lib.vdb_region_merge_f32(_ptr(eps), halves, bs, H, W, C, _ptr(oy), _ptr(ox), _ptr(cover_y), _ptr(cover_x), oy.numel(),
                                   ox.numel(), int(h), int(w), int(first), int(k), int(R), _ptr(masks), _ptr(out), _stream()),
          "region_merge")
    return out


def groupnorm(x1, gamma, beta, eps, act=ACT_NONE, x2=None, out=None, groups=32):
    """GN32(+SiLU) over NHWC bf16 [B,H,W,C1] (+ concat x2 [B,H,W,C2]) -> [B,H,W,C1+C2]."""
    _need(x1, BF16, "x1"); _need(x2, BF16, "x2"); _need(gamma, torch.float32, "gamma"); _need(beta, torch.float32, "beta")
    B = x1.shape[0]
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    HW = x1.numel() // (B * C1)
    if out is None:
        out = torch.empty(x1.shape[:-1] + (C1 + C2,), dtype=BF16, device=x1.device)
    partial = _gn_scratch(x1.device, lib.vdb_groupnorm_scratch_floats(B, HW))
    with _Span("groupnorm", 0.0, 2.0 * 3 * B * HW * (C1 + C2)):
        check(lib.vdb_groupnorm_nhwc(_ptr(x1), C1, _ptr(x2), C2, B, HW, groups, _ptr(gamma), _ptr(beta), float(eps),
                                     int(act), _ptr(partial), _ptr(out), _stream()), "groupnorm_nhwc")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    _need(x, BF16, "x"); _need(gamma, torch.float32, "gamma"); _need(beta, torch.float32, "beta")
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    with _Span("layernorm", 0.0, 2.0 * 2 * rows * C):
        check(lib.vdb_layernorm(_ptr(x), rows, C, _ptr(gamma), _ptr(beta), float(eps), _ptr(out), _stream()), "layernorm")
    return out


NORM_PLAN_FIELDS = ("family", "t0", "t1", "G", "S", "nsplit", "grid_x", "grid_y", "grid_z")
NORM_FAMILIES = {0: None, 1: "gn_bundle", 2: "gn_fused", 3: "gn_stats_apply", 4: "ln_rg", 5: "ln_warp"}


def norm_last_plan():
    """The kernel the last groupnorm / layernorm call on this thread launched (vdb_norm_last_plan): family (gn_bundle,
    gn_fused, gn_stats_apply, ln_rg, ln_warp), template parameters t0 / t1 (NVMAX / THREADS, NV, VPL / LPR, MAXV / R),
    GroupNorm's groups per CTA G, cluster size S and pixel splits nsplit, and the grid."""
    buf = (ctypes.c_int * len(NORM_PLAN_FIELDS))()
    n = lib.vdb_norm_last_plan(buf, len(buf))
    assert n == len(NORM_PLAN_FIELDS), n
    plan = dict(zip(NORM_PLAN_FIELDS, buf))
    plan["family"] = NORM_FAMILIES[plan["family"]]
    return plan


def affine_silu_rows(x, gamma, beta, act=ACT_SILU, out=None):
    """y[r, i] = act(x[r, i] * gamma[i] + beta[i]); x bf16 [rows, n], gamma / beta fp32 [n] (FCBlock's per-position GroupNorm affine)."""
    _need(x, BF16, "x"); _need(gamma, torch.float32, "gamma"); _need(beta, torch.float32, "beta")
    rows, n = x.shape
    if out is None:
        out = torch.empty_like(x)
    check(lib.vdb_affine_act_rows(_ptr(x), rows, n, _ptr(gamma), _ptr(beta), int(act), _ptr(out), _stream()), "affine_act_rows")
    return out


def pack_conv_weight(w, out=None, col0=0):
    """Conv2d weight fp32 [Cout, Cin, kh, kw] -> bf16 [Cout, ldo] with column col0 + (ky*kw + kx)*Cin + ci (C ABI repack)."""
    _need(w, torch.float32, "w")
    Cout, Cin, kh, kw = w.shape
    if out is None:
        out = torch.empty((Cout, col0 + kh * kw * Cin), dtype=BF16, device=w.device)
    check(lib.vdb_pack_conv_weight(_ptr(w), Cout, Cin, kh, kw, _ptr(out), out.stride(0), col0, _stream()), "pack_conv_weight")
    return out


def pack_geglu(w, b=None):
    """GEGLU.proj weight fp32 [2*n2, K] (+ bias) -> (bf16 rows interleaved per 256-row tile, fp32 bias in the same order)."""
    _need(w, torch.float32, "w")
    n2, K = w.shape[0] // 2, w.shape[1]
    wo = torch.empty((2 * n2, K), dtype=BF16, device=w.device)
    bo = torch.empty(2 * n2, dtype=torch.float32, device=w.device) if b is not None else None
    if b is not None:
        _need(b, torch.float32, "b")
    check(lib.vdb_pack_geglu(_ptr(w), _ptr(b) if b is not None else None, n2, K, _ptr(wo), _ptr(bo) if bo is not None else None,
                             _stream()), "pack_geglu")
    return wo, bo


def pad_heads(w, H, d, dpad):
    """attention projection fp32 [H*d, K] -> bf16 [H*dpad, K], zero rows after each head's d rows."""
    _need(w, torch.float32, "w")
    out = torch.empty((H * dpad, w.shape[1]), dtype=BF16, device=w.device)
    check(lib.vdb_pad_heads(_ptr(w), H, d, dpad, w.shape[1], _ptr(out), _stream()), "pad_heads")
    return out


def upsample2x(x, out=None):
    _need(x, BF16, "x")
    B, H, W, C = x.shape
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, C), dtype=BF16, device=x.device)
    check(lib.vdb_upsample2x_nhwc(_ptr(x), B, H, W, C, _ptr(out), _stream()), "upsample2x")
    return out


def upsample2x_conv3x3_folded(x, wf, bias=None):
    """nearest-2x upsample + 3x3 conv (pad 1) without materialising the upsampled image: four 2x2-tap convs on the source
    (one per output parity, weights folded by diffusion_utils.fold_upsample_conv3x3).
    x bf16 [B,H,W,C]; wf bf16 [4, N, 4*C] with N % 32 == 0; -> [B,2H,2W,N]."""
    B, H, W, _ = x.shape
    N = wf.shape[1]
    if N % 32:
        raise ValueError(f"upsample2x_conv3x3_folded: N = {N} is not a multiple of 32 (use upsample2x + conv3x3)")
    # modes 7..10: every parity conv stores straight into its pixels of the [B,2H,2W,N] result (output tensor map with
    # doubled strides): no interleave pass, no parity temporaries
    out = torch.empty((B, 2 * H, 2 * W, N), dtype=BF16, device=x.device)
    for par in range(4):
        conv3x3(x, wf[par], bias=bias, out=out, mode=7 + par, ksplit=1)
    return out


def im2col3x3_small(x, kpad=64, in_scale=1.0, in_shift=0.0, out=None):
    """x fp32 NHWC [B,H,W,Cin<=7] -> bf16 [B*H*W, kpad]."""
    _need(x, torch.float32, "x")
    B, H, W, Cin = x.shape
    if out is None:
        out = torch.empty((B * H * W, kpad), dtype=BF16, device=x.device)
    check(lib.vdb_im2col3x3_small(_ptr(x), B, H, W, Cin, kpad, float(in_scale), float(in_shift), _ptr(out), _stream()),
          "im2col3x3_small")
    return out


def nchw_to_nhwc(x, mul=1.0, add=0.0, out=None):
    _need(x, torch.float32, "x")
    B, C = x.shape[:2]
    HW = x.numel() // (B * C)
    if out is None:
        out = torch.empty((B,) + tuple(x.shape[2:]) + (C,), dtype=torch.float32, device=x.device)
    check(lib.vdb_permute_f32(_ptr(x), B, C, HW, 1, float(mul), float(add), 0, _ptr(out), _stream()), "permute")
    return out


def nhwc_to_nchw(x, mul=1.0, add=0.0, clamp01=False, out=None):
    _need(x, torch.float32, "x")
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    if out is None:
        out = torch.empty((B, C) + tuple(x.shape[1:-1]), dtype=torch.float32, device=x.device)
    check(lib.vdb_permute_f32(_ptr(x), B, C, HW, 0, float(mul), float(add), 1 if clamp01 else 0, _ptr(out), _stream()),
          "permute")
    return out


def to_bf16(x, out=None):
    _need(x, torch.float32, "x"); _need(out, BF16, "out")
    _same_shape(x, out, "out")
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    check(lib.vdb_cast_f32_bf16(_ptr(x), _ptr(out), x.numel(), _stream()), "cast")
    return out


def to_f32(x, out=None):
    _need(x, BF16, "x"); _need(out, torch.float32, "out")
    _same_shape(x, out, "out")
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    check(lib.vdb_cast_bf16_f32(_ptr(x), _ptr(out), x.numel(), _stream()), "cast")
    return out


def pointwise_small(x, w, bias=None, pre_mul=1.0, out=None):
    """x fp32 [..., Cin<=8] NHWC, w fp32 [Cout, Cin] -> fp32 [..., Cout]."""
    _need(x, torch.float32, "x"); _need(w, torch.float32, "w"); _need(bias, torch.float32, "bias")
    _need(out, torch.float32, "out")
    if w.dim() != 2:
        raise ValueError(f"w: expected [Cout, Cin], got {tuple(w.shape)}")
    cout, cin = w.shape
    if x.dim() < 1 or x.shape[-1] != cin:
        raise ValueError(f"x: expected [..., {cin}] for w {tuple(w.shape)}, got {tuple(x.shape)}")
    if bias is not None and bias.numel() != cout:
        raise ValueError(f"bias: expected {cout} elements, got {bias.numel()}")
    npix = x.numel() // cin
    if out is None:
        out = torch.empty(x.shape[:-1] + (cout,), dtype=torch.float32, device=x.device)
    if out.numel() != npix * cout:
        raise ValueError(f"out: expected {npix * cout} elements ({tuple(x.shape[:-1]) + (cout,)}), got {tuple(out.shape)}")
    check(lib.vdb_pointwise_small(_ptr(x), npix, cin, cout, _ptr(w), _ptr(bias), float(pre_mul), _ptr(out), _stream()),
          "pointwise_small")
    return out


def gaussian_sample(moments, noise=None, post_mul=1.0, out=None):
    """moments fp32 NHWC [..., 2C]; noise fp32 NHWC [..., C] or None (posterior mean)."""
    _need(moments, torch.float32, "moments"); _need(noise, torch.float32, "noise"); _need(out, torch.float32, "out")
    if moments.dim() < 1 or moments.shape[-1] < 2 or moments.shape[-1] % 2:
        raise ValueError(f"moments: expected [..., 2C] (mean | logvar), got {tuple(moments.shape)}")
    C = moments.shape[-1] // 2
    npix = moments.numel() // (2 * C)
    shape = moments.shape[:-1] + (C,)
    if noise is not None and noise.shape != shape:
        raise ValueError(f"noise: expected {tuple(shape)}, got {tuple(noise.shape)}")
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=moments.device)
    if out.numel() != npix * C:
        raise ValueError(f"out: expected {tuple(shape)}, got {tuple(out.shape)}")
    check(lib.vdb_gaussian_sample(_ptr(moments), _ptr(noise), C, npix, float(post_mul), _ptr(out), _stream()),
          "gaussian_sample")
    return out


def timestep_embedding(ts, dim, max_period=10000, step_idx=None, batch=None, out=None):
    """ts int64 device tensor [B] (or a table + step_idx int32 device scalar, broadcast to `batch` rows)."""
    _need(ts, torch.int64, "timesteps"); _need(step_idx, torch.int32, "step_idx"); _need(out, torch.float32, "out")
    B = batch if step_idx is not None else ts.shape[0]
    if out is None:
        out = torch.empty((B, dim), dtype=torch.float32, device=ts.device)
    if out.numel() != B * dim:
        raise ValueError(f"out: expected ({B}, {dim}), got {tuple(out.shape)}")
    nlp = torch.tensor(-math.log(max_period), dtype=torch.float32).item()
    check(lib.vdb_timestep_embedding(_ptr(ts), _ptr(step_idx), B, dim, nlp, _ptr(out), _stream()), "timestep_embedding")
    return out


def linear_small(x, w, bias=None, act_in=ACT_NONE, act_out=ACT_NONE, out=None):
    """x fp32 [M<=16,K], w bf16 [N,K] -> fp32 [M,N]."""
    _need(x, torch.float32, "x"); _need(w, BF16, "w"); _need(bias, torch.float32, "bias"); _need(out, torch.float32, "out")
    if x.dim() != 2 or w.dim() != 2 or w.shape[1] != x.shape[1]:
        raise ValueError(f"w: expected [N, {x.shape[-1]}] for x {tuple(x.shape)}, got {tuple(w.shape)}")
    M, K = x.shape
    N = w.shape[0]
    if bias is not None and bias.numel() != N:
        raise ValueError(f"bias: expected {N} elements, got {bias.numel()}")
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    if out.shape != (M, N):
        raise ValueError(f"out: expected ({M}, {N}), got {tuple(out.shape)}")
    check(lib.vdb_linear_small(_ptr(x), M, K, _ptr(w), N, _ptr(bias), int(act_in), int(act_out), _ptr(out), _stream()),
          "linear_small")
    return out


def softmax_rows(x, scale=1.0, out=None):
    """Row softmax of bf16 [..., n] (x * scale) -> bf16 of the same shape and strides (the kernel walks both with x's row stride)."""
    _need(x, BF16, "x"); _need(out, BF16, "out")
    n = x.shape[-1]
    rows = x.numel() // n
    if out is None:
        out = torch.empty_like(x)
    if out.shape != x.shape or out.stride() != x.stride():
        raise ValueError(f"out: expected shape {tuple(x.shape)} with strides {x.stride()}, got {tuple(out.shape)} with {out.stride()}")
    check(lib.vdb_softmax_rows(_ptr(x), rows, n, x.stride(-2) if x.dim() > 1 else n, float(scale), _ptr(out), _stream()),
          "softmax_rows")
    return out


def to_uint8_hwc(images):
    """fp32 CUDA [n,3,H,W] in [0,1] -> uint8 [n,H,W,3] with torchvision.ToPILImage semantics (x * 255 truncated)."""
    _need(images, torch.float32, "images")
    n, ch, H, W = images.shape
    assert ch == 3
    out = torch.empty((n, H, W, 3), dtype=torch.uint8, device=images.device)
    check(lib.vdb_clip_to_u8_hwc(_ptr(images), n, H, W, _ptr(out), _stream()), "clip_to_u8_hwc")
    return out


def clip_preprocess_device(images, tables, size, mean, std):
    """images fp32 CUDA [n,3,H,W] in [0,1] -> fp32 [n,3,size,size], bit-exact with ToPILImage + Pillow bicubic resize of the
    shortest side + centre crop + rescale + normalise (reference clip.py:88-94 runs this on the host through PIL).
    tables = {"nw","nh","h": (bounds, kk) or None, "v": (bounds, kk) or None} with int32 CUDA tensors (clip.pil_bicubic_coeffs)."""
    import ctypes
    _need(images, torch.float32, "images")
    n, _, H, W = images.shape
    nw, nh = tables["nw"], tables["nh"]
    u8 = torch.empty((n, H, W, 3), dtype=torch.uint8, device=images.device)
    check(lib.vdb_clip_to_u8_hwc(_ptr(images), n, H, W, _ptr(u8), _stream()), "clip_to_u8_hwc")
    if tables["h"] is not None:
        hb, hk = tables["h"]
        mid = torch.empty((n, H, nw, 3), dtype=torch.uint8, device=images.device)
        check(lib.vdb_resample_h_u8(_ptr(u8), n, H, W, nw, _ptr(hb), _ptr(hk), hk.shape[1], _ptr(mid), _stream()), "resample_h_u8")
    else:
        mid = u8
    out = torch.empty((n, 3, size, size), dtype=torch.float32, device=images.device)
    vb, vk = tables["v"] if tables["v"] is not None else (None, None)
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    check(lib.vdb_resample_v_crop_norm(_ptr(mid), n, H, nw, _ptr(vb), _ptr(vk), 0 if vk is None else vk.shape[1],
                                       (nh - size) // 2, (nw - size) // 2, size, m3, s3, _ptr(out), _stream()),
          "resample_v_crop_norm")
    return out


# ------------------------------------------------------------------------------------------------ CLIP ends
def clip_text_embed(tokens, tok_emb, pos_emb, Lp):
    _need(tokens, torch.int64, "tokens"); _need(tok_emb, torch.float32, "tok_emb"); _need(pos_emb, torch.float32, "pos_emb")
    B, L = tokens.shape
    C = tok_emb.shape[1]
    if pos_emb.dim() != 2 or pos_emb.shape[0] < L or pos_emb.shape[1] != C:
        raise ValueError(f"pos_emb: expected [>= {L}, {C}], got {tuple(pos_emb.shape)}")
    x = torch.empty((B, Lp, C), dtype=BF16, device=tokens.device)
    check(lib.vdb_clip_text_embed(_ptr(tokens), _ptr(tok_emb), _ptr(pos_emb), B, L, Lp, C, _ptr(x), _stream()), "clip_text_embed")
    return x


def patchify(pixels, patch, kpad):
    _need(pixels, torch.float32, "pixels")
    B, Cin, H, W = pixels.shape
    assert H == W
    g = H // patch
    y = torch.empty((B * g * g, kpad), dtype=BF16, device=pixels.device)
    check(lib.vdb_patchify(_ptr(pixels), B, Cin, H, patch, kpad, _ptr(y), _stream()), "patchify")
    return y


def vit_assemble(patches, cls, pos, B, L, Lp, tok_scale=None):
    _need(patches, BF16, "patches"); _need(cls, torch.float32, "cls"); _need(pos, torch.float32, "pos")
    _need(tok_scale, torch.float32, "tok_scale")
    C = patches.shape[1]
    if patches.dim() != 2 or patches.shape[0] != B * (L - 1):
        raise ValueError(f"patches: expected [{B * (L - 1)}, C] (B * (L - 1) rows), got {tuple(patches.shape)}")
    if cls.numel() != C:
        raise ValueError(f"cls: expected {C} elements, got {cls.numel()}")
    if pos.dim() != 2 or pos.shape[0] < L or pos.shape[1] != C:
        raise ValueError(f"pos: expected [>= {L}, {C}], got {tuple(pos.shape)}")
    if tok_scale is not None and tok_scale.numel() != B * L:
        raise ValueError(f"tok_scale: expected {B * L} elements ([{B}, {L}]), got {tuple(tok_scale.shape)}")
    x = torch.empty((B, Lp, C), dtype=BF16, device=patches.device)
    check(lib.vdb_vit_assemble(_ptr(patches), _ptr(cls), _ptr(pos), _ptr(tok_scale), B, L, Lp, C, _ptr(x), _stream()), "vit_assemble")
    return x


def scale_by_row_norm(z, L, idx=None, row_scale=None):
    """z bf16 [B, Lp, C] -> fp32 [B, L, C] divided by the norm of row idx[b] (token 0 when idx is None)."""
    _need(z, BF16, "z"); _need(idx, torch.int32, "idx"); _need(row_scale, torch.float32, "row_scale")
    B, Lp, C = z.shape
    if idx is not None and idx.numel() != B:
        raise ValueError(f"idx: expected {B} elements, got {idx.numel()}")
    if row_scale is not None and row_scale.numel() != B * L:
        raise ValueError(f"row_scale: expected {B * L} elements ([{B}, {L}]), got {tuple(row_scale.shape)}")
    out = torch.empty((B, L, C), dtype=torch.float32, device=z.device)
    check(lib.vdb_scale_by_row_norm(_ptr(z), _ptr(idx), _ptr(row_scale), B, L, Lp, C, _ptr(out), _stream()), "scale_by_row_norm")
    return out


# ------------------------------------------------------------------------------------------------
# Optimus GPT-2 text decoder (optimus.py:662-688, 746-763): one token step for R <= 16 rows
# ------------------------------------------------------------------------------------------------
ACT_GELU_TANH = 5
ACT_TANH = 6            # BertPooler (textdec_gemv only)


def textdec_gemv(x, w, out, bias=None, ln=None, act=ACT_NONE, accumulate=False):
    """out[R,N] (=|+=) act(LN(x) @ w^T + bias); x fp32 [R<=16, K] (row-strided ok), w bf16 [N, K], ln = (gamma, beta, eps) or None."""
    _need(x, torch.float32, "x", rows_ok=True); _need(w, BF16, "w", rows_ok=True); _need(out, torch.float32, "out", rows_ok=True)
    _need(bias, torch.float32, "bias")
    g, b, eps = ln if ln is not None else (None, None, 0.0)
    _need(g, torch.float32, "ln_gamma"); _need(b, torch.float32, "ln_beta")
    R, K = x.shape
    N = w.shape[0]
    check(lib.vdb_textdec_gemv(_ptr(x), R, K, x.stride(0), _ptr(g), _ptr(b), float(eps), _ptr(w), N, w.stride(0), _ptr(bias),
                               int(act), int(bool(accumulate)), _ptr(out), out.stride(0), _stream()), "textdec_gemv")
    return out


def textdec_attention(qkv, mem, kcache, vcache, step, out, scale=0.125, src=None):
    """qkv fp32 [R, 3*H*64], mem fp32 [R, >=H*64] (this layer's latent slice), caches fp32 [R, H, T, 64], step int32 [1].
    src int32 [R, T] (beam search): cache slot j of row r is read from physical row src[r, j] (see vdb_textdec_attention)."""
    for n, t in (("qkv", qkv), ("mem", mem), ("out", out)):
        _need(t, torch.float32, n, rows_ok=True)
    _need(kcache, torch.float32, "kcache"); _need(vcache, torch.float32, "vcache"); _need(step, torch.int32, "step")
    _need(src, torch.int32, "src")
    R, H, T, _ = kcache.shape
    if src is not None and tuple(src.shape) != (R, T):
        raise ValueError(f"textdec_attention: src must be [{R}, {T}], got {list(src.shape)}")
    check(lib.vdb_textdec_attention(_ptr(qkv), qkv.stride(0), _ptr(mem), mem.stride(0), _ptr(kcache), _ptr(vcache), _ptr(src), R, H,
                                    T, _ptr(step), float(scale), _ptr(out), out.stride(0), _stream()), "textdec_attention")
    return out


def textdec_embed(tokens, step, wte, wpe, emb, out, pos_offset=1):
    """out[r] = wte[tokens[r, *step]] + wpe[*step + pos_offset] + emb[r]; tokens int32 [R, L], tables / emb / out fp32."""
    _need(tokens, torch.int32, "tokens"); _need(step, torch.int32, "step")
    for n, t in (("wte", wte), ("wpe", wpe), ("emb", emb), ("out", out)):
        _need(t, torch.float32, n)
    R, D = out.shape
    check(lib.vdb_textdec_embed(_ptr(tokens), tokens.stride(0), _ptr(step), _ptr(wte), wte.shape[0], _ptr(wpe), wpe.shape[0],
                                int(pos_offset), _ptr(emb), R, D, _ptr(out), _stream()), "textdec_embed")
    return out


def textdec_sample(logits, tokens, done, lengths, step, temperature=1.0, seed=None, uniforms=None, forced=None, eos=50259,
                   max_len=30, record=None, top_k=0, top_p=0.0):
    """Token *step+1 of every unfinished row ~ softmax(logits / temperature) (see vdb_textdec_sample).  seed: device uint64 [1]
    (as int64), uniforms: fp64 [R, >=steps] given draws, forced: int32 [R, L] teacher-forced tokens, record: fp32 [steps, R, V].
    top_k > 0 or 0 < top_p < 1 draw from the tokens those cuts keep instead."""
    _need(logits, torch.float32, "logits", rows_ok=True)
    _need(tokens, torch.int32, "tokens"); _need(done, torch.int32, "done"); _need(lengths, torch.int32, "lengths")
    _need(step, torch.int32, "step"); _need(seed, torch.int64, "seed"); _need(uniforms, torch.float64, "uniforms")
    _need(forced, torch.int32, "forced"); _need(record, torch.float32, "record")
    R, V = logits.shape
    check(lib.vdb_textdec_sample(_ptr(logits), R, V, logits.stride(0), float(temperature), int(top_k), float(top_p), _ptr(seed),
                                 _ptr(uniforms), uniforms.stride(0) if uniforms is not None else 0, _ptr(forced),
                                 forced.stride(0) if forced is not None else 0, _ptr(tokens), tokens.stride(0), _ptr(done),
                                 _ptr(lengths), _ptr(step), int(eos), int(max_len), _ptr(record), _stream()), "textdec_sample")


def textdec_beam_step(logits, num_beams, tokens, src, scores, done, lengths, step, cand_tok, cand_logp, temperature=1.0,
                      eos=50259, max_len=30, record=None, trace=None):
    """One beam-search step over rows r = latent * num_beams + beam (see vdb_textdec_beam_step): tokens int32 [R, L], src int32
    [R, T], scores fp64 [R], done / lengths int32 [R]; cand_tok int32 / cand_logp fp64 with >= R * num_beams elements (scratch);
    record fp32 [steps, R, V], trace fp64 [steps, R, 3] (parent beam, token or -1, score)."""
    _need(logits, torch.float32, "logits", rows_ok=True)
    for n, t in (("tokens", tokens), ("src", src), ("done", done), ("lengths", lengths), ("step", step), ("cand_tok", cand_tok)):
        _need(t, torch.int32, n)
    _need(scores, torch.float64, "scores"); _need(cand_logp, torch.float64, "cand_logp")
    _need(record, torch.float32, "record"); _need(trace, torch.float64, "trace")
    R, V = logits.shape
    if cand_tok.numel() < R * num_beams or cand_logp.numel() < R * num_beams:
        raise ValueError(f"textdec_beam_step: the candidate buffers need {R * num_beams} elements")
    check(lib.vdb_textdec_beam_step(_ptr(logits), R, V, logits.stride(0), float(temperature), int(num_beams), _ptr(tokens),
                                    tokens.stride(0), _ptr(src), src.stride(0), _ptr(scores), _ptr(done), _ptr(lengths), _ptr(step),
                                    int(eos), int(max_len), _ptr(cand_tok), _ptr(cand_logp), _ptr(record), _ptr(trace), _stream()),
          "textdec_beam_step")


def textdec_repetition(logits, tokens, done, step, penalty=1.0, ngram=0):
    """The repetition penalty and no-repeat n-gram bans on logits fp32 [R, V] in place (see vdb_textdec_repetition): row r's
    history is tokens[r, :*step + 1] (int32 [R, L]); rows with done[r] != 0 are left as they are.  penalty 1 and ngram 0
    launch nothing."""
    _need(logits, torch.float32, "logits", rows_ok=True)
    _need(tokens, torch.int32, "tokens"); _need(done, torch.int32, "done"); _need(step, torch.int32, "step")
    R, V = logits.shape
    check(lib.vdb_textdec_repetition(_ptr(logits), R, V, logits.stride(0), _ptr(tokens), tokens.stride(0), _ptr(done), _ptr(step),
                                     float(penalty), int(ngram), _stream()), "textdec_repetition")
    return logits


# ------------------------------------------------------------------------------------------------
# Semantic/style disentanglement (app.py:48-127): the rank adjustment of the image context, one launch
# ------------------------------------------------------------------------------------------------
def rank_adjust(x, factors, keep_remainder, R, niter=100, out=None, s_out=None, u_out=None, v_out=None):
    """x fp32 [n, m, 768] -> x_new (see vdb_rank_adjust_f32): the rank-q PCA of each item's row-centred x, started from R fp32
    [m, q] (shared by all items), with S scaled by factors fp32 [q]; keep_remainder adds back what the rank-q part misses.
    Optional outputs: s_out fp32 [n, q] the unscaled S, u_out [n, m, q] and v_out [n, 768, q] the factors U and V."""
    for name, t in (("x", x), ("factors", factors), ("R", R), ("s_out", s_out), ("u_out", u_out), ("v_out", v_out)):
        _need(t, torch.float32, name)
    if x.dim() != 3 or R.dim() != 2 or R.shape[0] != x.shape[1] or factors.numel() != R.shape[1]:
        raise ValueError(f"rank_adjust: x {tuple(x.shape)}, R {tuple(R.shape)} and factors {tuple(factors.shape)} disagree")
    n, m, d = x.shape
    q = R.shape[1]
    if out is None:
        out = torch.empty_like(x)
    _need(out, torch.float32, "out")
    if out.shape != x.shape:
        raise ValueError(f"rank_adjust: out must be {list(x.shape)}, got {list(out.shape)}")
    x0, o0, nbytes = x.data_ptr(), out.data_ptr(), x.numel() * 4    # both contiguous fp32 of the same size
    if o0 < x0 + nbytes and x0 < o0 + nbytes:
        raise ValueError("rank_adjust: out must not overlap x (an out shifted against x writes rows another item has yet to read)")
    for name, t, shape in (("s_out", s_out, (n, q)), ("u_out", u_out, (n, m, q)), ("v_out", v_out, (n, d, q))):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError(f"rank_adjust: {name} must be {list(shape)}, got {list(t.shape)}")
    check(lib.vdb_rank_adjust_f32(_ptr(x), n, m, d, _ptr(R), q, int(niter), _ptr(factors), int(bool(keep_remainder)), _ptr(out),
                                  _ptr(s_out), _ptr(u_out), _ptr(v_out), _stream()), "rank_adjust")
    return out
