"""SpatialTransformer / BasicTransformerBlock / CrossAttention / GEGLU feed-forward on vdb200 kernels
(reference lib/model_zoo/attention.py:37-64, 152-266).  Same constructor signatures and parameter
names; activations are NHWC bf16 (the reference's 'b c h w -> b (h w) c' rearrange is a no-op here).

Kernel schedule of one SpatialTransformer (x: [B,H,W,C] bf16):
  GN32(eps 1e-6) -> proj_in GEMM -> [LN -> fused q|k GEMM + V^T GEMM -> flash attention -> to_out GEMM(+resid)]
  -> [LN -> q GEMM (K, V^T of the context cached across DDIM steps) -> flash attention -> to_out GEMM(+resid)]
  -> LN -> GEGLU GEMM -> FF-out GEMM(+resid) -> proj_out GEMM (+ x_in, * mixing ratio)
The three LayerNorms are not kernels where the token grid allows it (ln_fold_fits): gamma is folded into the weights of the GEMMs that
consume the normalised tokens, mean / rstd arrive as per-32-channel partial sums written by the epilogue of the GEMM that PRODUCED
the tokens (proj_in, the two to_out), and the consumer applies r * (x W'^T - mu * s) + c in its own epilogue (vdb_gemm_ln_bf16).
"""
import torch
from torch import nn

from .diffusion_utils import PackedModule, bf16, f32, require_cuda, zero_module, pack_conv1x1


def _ops():
    from vdb200 import ops
    return ops


class PaddedContext(object):
    """A context batch already in kernel layout: bf16 [B, Lp, C] with Lp = L rounded up to 8 and zero pad rows.
    DDIMSampler keeps one per context in a persistent buffer so the captured CUDA graph (and the cached K / V^T
    of every cross-attention layer) stay valid when a new prompt is copied in.  edit: the prompt_edit.EditState of a
    Prompt-to-Prompt walk on this context (its rows past the batch's are the edited contexts), else None."""

    def __init__(self, data, length, edit=None):
        self.data, self.length, self.edit = data, length, edit


class KeyMass(object):
    """Where the mid block's self-attention adds its per-key attention mass for self-attention guidance (lib/model_zoo/sag.py):
    mass fp32 [n, N] for batch items row0 .. row0 + n - 1, each head's column sums weighted by ratio / heads."""

    def __init__(self, mass, row0=0, ratio=1.0):
        self.mass, self.row0, self.ratio = mass, row0, ratio

    def weighted(self, ratio):
        return KeyMass(self.mass, self.row0, ratio)


def ln_fold_fits(inner, B, H, W):
    """LayerNorms folded into the neighbouring GEMMs need their TMA-store epilogues: inner % 32 == 0, and the B * H * W tokens
    are the N of the V^T projection.  Other token grids run the LayerNorm kernels."""
    return inner % 32 == 0 and (H * W) % 8 == 0 and (B * H * W) % 32 == 0


def fold_layernorm(w, b, gamma, beta):
    """Linear(LayerNorm(x)) = r * (x W'^T - mu * s) + c  ->  (W' bf16 [N,K], s fp32 [N], c fp32 [N])  (include/vdb200.h)."""
    wf = w.detach().float()
    wg = (wf * gamma.detach().float()[None, :]).to(torch.bfloat16).contiguous()
    s = wg.float().sum(1).contiguous()                      # of the ROUNDED weights: what the tensor core multiplies mu with
    c = wf @ beta.detach().float()
    if b is not None:
        c = c + b.detach().float()
    return wg, s, c.contiguous()


def Normalize(in_channels):
    return torch.nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class GEGLU(PackedModule):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def _pack(self):
        ops = _ops()
        w, b = self.proj.weight, self.proj.bias
        n2 = w.shape[0] // 2
        half = 128  # per 256-column tile: 128 value rows then their 128 gate rows
        if n2 % half:
            raise ValueError("GEGLU width must be a multiple of 128 for the fused epilogue")
        idx = []
        for t in range(n2 // half):
            idx += list(range(t * half, (t + 1) * half)) + list(range(n2 + t * half, n2 + (t + 1) * half))
        idx = torch.tensor(idx, device=w.device)
        return {"w": bf16(w.detach()[idx]), "b": f32(b.detach()[idx]), "act": ops.ACT_GEGLU, "idx": idx}

    def forward(self, x):  # x: [rows, C] bf16
        p = self.packed()
        return _ops().gemm(x, p["w"], bias=p["b"], act=p["act"])


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.):
        super().__init__()
        if not glu:
            raise NotImplementedError("only the gated (GEGLU) feed-forward is on the VD hot path")
        inner_dim = int(dim * mult)
        dim_out = dim if dim_out is None else dim_out
        self.net = nn.Sequential(GEGLU(dim, inner_dim), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out))


class CrossAttention(PackedModule):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.):
        super().__init__()
        inner_dim = dim_head * heads
        self.is_self = context_dim is None
        context_dim = query_dim if context_dim is None else context_dim
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))
        self._kv_cache = None

    def _pad_heads(self, w, dpad):
        """[H*d, K] -> [H*dpad, K] with zero rows after each head's d rows"""
        h, d = self.heads, self.dim_head
        out = torch.zeros(h, dpad, w.shape[1], dtype=torch.bfloat16, device=w.device)
        out[:, :d] = w.detach().view(h, d, -1).to(torch.bfloat16)
        return out.view(h * dpad, -1).contiguous()

    def _pad_head_vec(self, v, dpad):
        h, d = self.heads, self.dim_head
        out = torch.zeros(h, dpad, dtype=torch.float32, device=v.device)
        out[:, :d] = v.view(h, d)
        return out.view(-1).contiguous()

    def pack_folded(self, gamma, beta):
        """the projections that read LayerNorm(x), with that LayerNorm folded in (fold_layernorm), heads padded as in _pack"""
        dk, dv = _ops().attention_pads(self.dim_head)
        wq, sq, cq = fold_layernorm(self.to_q.weight, None, gamma, beta)
        out = {"wq": self._pad_heads(wq, dk), "sq": self._pad_head_vec(sq, dk), "cq": self._pad_head_vec(cq, dk)}
        if self.is_self:
            wk, sk, ck = fold_layernorm(self.to_k.weight, None, gamma, beta)
            wv, sv, cv = fold_layernorm(self.to_v.weight, None, gamma, beta)
            out.update({"wqk": torch.cat([out["wq"], self._pad_heads(wk, dk)], 0).contiguous(),
                        "sqk": torch.cat([out["sq"], self._pad_head_vec(sk, dk)]).contiguous(),
                        "cqk": torch.cat([out["cq"], self._pad_head_vec(ck, dk)]).contiguous(),
                        "wv": self._pad_heads(wv, dv), "sv": self._pad_head_vec(sv, dv), "cv": self._pad_head_vec(cv, dv)})
        return out

    def _pack(self):
        dk, dv = _ops().attention_pads(self.dim_head)
        wq, wk = self._pad_heads(self.to_q.weight, dk), self._pad_heads(self.to_k.weight, dk)
        self._kv_cache = None
        return {"dk": dk, "dv": dv, "wq": wq, "wk": wk, "wqk": torch.cat([wq, wk], 0).contiguous() if self.is_self else None,
                "wv": self._pad_heads(self.to_v.weight, dv), "wo": bf16(self.to_out[0].weight),
                "bo": f32(self.to_out[0].bias)}

    _KV_CACHE_SLOTS = 4

    def _kv_get(self, key):
        for ent in (self._kv_cache or ()):
            if ent[0] == key:
                return ent
        return None

    def _kv_put(self, ent):
        """small per-layer cache keyed by the context buffer: two contexts of the same type (sample_multicontext with two
        'image' c_infos) or two samplers sharing one model keep their own K / V^T buffers instead of evicting each other
        (which silently re-projected the context inside every step and forced a graph re-capture per sample() call)"""
        cache = [e for e in (self._kv_cache or ()) if e[0] != ent[0]]
        cache.append(ent)
        self._kv_cache = cache[-self._KV_CACHE_SLOTS:]

    def context_kv(self, context):
        """K [B*Lp, H*dk] and V^T [H*dvp, B*Lp] of a context; cached while the same tensor (and version) is passed
        again — the context is constant over the DDIM loop, so this runs once per sample() call, not per step."""
        p = self.packed()
        ops = _ops()
        if isinstance(context, PaddedContext):
            data, L = context.data, context.length
            B, Lp, Cc = data.shape
            key = ("padded", data.data_ptr(), (B, Lp, Cc), L)
            cflat = data.view(B * Lp, Cc)
            ent = self._kv_get(key)
            if ent is not None:
                k, vt, ver = ent[1]
                if ver != data._version:          # new prompt copied into the same buffer: refresh IN PLACE
                    ops.gemm(cflat, p["wk"], out=k)
                    ops.gemm(p["wv"], cflat, out=vt)
                    self._kv_put((key, (k, vt, data._version), data))
                return k, vt, L, Lp
            k = ops.gemm(cflat, p["wk"])
            vt = ops.gemm(p["wv"], cflat)
            self._kv_put((key, (k, vt, data._version), data))
            return k, vt, L, Lp
        # the cache entry HOLDS the context tensor: while it is alive no other allocation can reuse its address, so
        # (pointer, version, shape) identifies the contents (a freed-and-reallocated buffer would otherwise alias it)
        key = (context.data_ptr(), context._version, tuple(context.shape), context.dtype)
        ent = self._kv_get(key)
        if ent is not None:
            return ent[1]
        B, L, Cc = context.shape
        Lp = (L + 7) // 8 * 8   # kv stride per batch item must be a multiple of 8 (TMA alignment)
        cpad = torch.zeros(B, Lp, Cc, dtype=torch.bfloat16, device=context.device)
        cpad[:, :L] = context.to(torch.bfloat16)
        cflat = cpad.view(B * Lp, Cc)
        val = (ops.gemm(cflat, p["wk"]), ops.gemm(p["wv"], cflat), L, Lp)
        self._kv_put((key, val, context))
        return val

    def _attend(self, q, k, vt, o, B, N, Nk, edit, cross, q_col0=0, k_col0=0, kv_bstride=0, key_mass=None):
        """The layer's flash attention.  Under a prompt edit (lib/model_zoo/prompt_edit.py) the indexed form with the edit's
        table for this layer, the refinement's accumulating second term, and the word maps at the 1/4-side cross layers.
        key_mass: a KeyMass of a self-attention layer, which also receives its key mass from the same q and k."""
        ops = _ops()
        H, d = self.heads, self.dim_head
        items = None if edit is None else edit.items(cross, N)
        kw = dict(scale=self.scale, q_col0=q_col0, k_col0=k_col0, kv_bstride=kv_bstride)
        if items is None:
            ops.attention(q, k, vt, o, B, H, N, Nk, d, **kw)
            if key_mass is not None:
                ops.sattn_key_mass(q, k, key_mass.mass, key_mass.row0, H, N, d, w=key_mass.ratio / H, **kw)
            return
        Bkv = edit.ctx_batch if cross else B
        ops.attention(q, k, vt, o, B, H, N, Nk, d, items=items, step_idx=edit.idx, Bkv=Bkv, **kw)
        if cross and edit.cross2 is not None:
            ops.attention(q, k, vt, o, B, H, N, Nk, d, items=edit.cross2, step_idx=edit.idx, Bkv=Bkv, accumulate=True, **kw)
        if cross and edit.maps_at(N):
            ops.xattn_word_map(q, k, edit.w, edit.map, edit.c0, H, N, Nk, d, kv_bstride=kv_bstride, scale=self.scale)

    def forward(self, x, context=None, resid=None, B=1, edit=None, key_mass=None):
        """x: [B*N, C] bf16 (already layer-normed); returns to_out(attn) + resid as [B*N, C] bf16.  edit: the prompt edit of a
        self-attention layer (a cross-attention layer reads it from its context).  key_mass: see _attend."""
        ops = _ops()
        p = self.packed()
        H, d, dk = self.heads, self.dim_head, p["dk"]
        N = x.shape[0] // B
        o = torch.empty(x.shape[0], H * d, dtype=torch.bfloat16, device=x.device)
        if context is None and N % 8 == 0:
            qk = ops.gemm(x, p["wqk"])                    # [B*N, 2*H*dk]: q | k
            vt = ops.gemm(p["wv"], x)                     # [H*dvp, B*N]
            self._attend(qk, qk, vt, o, B, N, N, edit, False, q_col0=0, k_col0=H * dk, key_mass=key_mass)
        elif context is None:
            # ragged token count (latent sides not a multiple of 8 at this level): keys/values from a copy of
            # the tokens padded to a multiple of 8 per batch item (TMA alignment of the V^T columns)
            Np = (N + 7) // 8 * 8
            xp = torch.zeros(B, Np, x.shape[1], dtype=torch.bfloat16, device=x.device)
            xp[:, :N] = x.view(B, N, -1)
            xp = xp.view(B * Np, -1)
            q = ops.gemm(x, p["wq"])
            k = ops.gemm(xp, p["wk"])
            vt = ops.gemm(p["wv"], xp)
            self._attend(q, k, vt, o, B, N, N, edit, False, kv_bstride=Np, key_mass=key_mass)
        else:
            q = ops.gemm(x, p["wq"])
            k, vt, L, Lp = self.context_kv(context)
            self._attend(q, k, vt, o, B, N, L, getattr(context, "edit", None), True, kv_bstride=Lp)
        return ops.gemm(o, p["wo"], bias=p["bo"], resid=resid)

    def forward_folded(self, x, ln, fp, context=None, resid=None, B=1, stats_out=None, edit=None, key_mass=None):
        """x: [B*N, C] bf16 RAW tokens, ln: ops.LnFold with their LayerNorm statistics, fp: pack_folded(); to_out writes the
        statistics of ITS output rows into stats_out (the next LayerNorm's input).  Self-attention needs N % 8 == 0."""
        ops = _ops()
        p = self.packed()
        H, d, dk = self.heads, self.dim_head, p["dk"]
        N = x.shape[0] // B
        o = torch.empty(x.shape[0], H * d, dtype=torch.bfloat16, device=x.device)
        if context is None:
            qk = ops.gemm_ln(x, fp["wqk"], bias=fp["cqk"], ln=ln, colsum=fp["sqk"])                       # [B*N, 2*H*dk]: q | k
            vt = ops.gemm_ln(fp["wv"], x, ln=ln, colsum=fp["sv"], on_cols=True, rowbias=fp["cv"])       # [H*dvp, B*N]
            self._attend(qk, qk, vt, o, B, N, N, edit, False, q_col0=0, k_col0=H * dk, key_mass=key_mass)
        else:
            q = ops.gemm_ln(x, fp["wq"], bias=fp["cq"], ln=ln, colsum=fp["sq"])
            k, vt, L, Lp = self.context_kv(context)
            self._attend(q, k, vt, o, B, N, L, getattr(context, "edit", None), True, kv_bstride=Lp)
        if stats_out is None:
            return ops.gemm(o, p["wo"], bias=p["bo"], resid=resid)
        return ops.gemm_ln(o, p["wo"], bias=p["bo"], resid=resid, stats_out=stats_out)      # -> (tokens, partials per row)


class BasicTransformerBlock(PackedModule):
    def __init__(self, dim, n_heads, d_head, dropout=0., context_dim=None, gated_ff=True, checkpoint=True,
                 disable_self_attn=False):
        super().__init__()
        if disable_self_attn:
            raise NotImplementedError("disable_self_attn=True is not used by the VD configs")
        self.disable_self_attn = disable_self_attn
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.norm3 = nn.LayerNorm(dim)
        self.checkpoint = checkpoint

    def _pack(self):
        out = {n: (f32(getattr(self, n).weight), f32(getattr(self, n).bias)) for n in ("norm1", "norm2", "norm3")} | \
            {"w2": bf16(self.ff.net[2].weight), "b2": f32(self.ff.net[2].bias)}
        if self.norm1.weight.shape[0] % 32 == 0:
            g = self.ff.net[0]
            idx = g.packed()["idx"]                          # GEGLU row order (value / gate halves per 256-column tile)
            wf, sf, cf = fold_layernorm(g.proj.weight, g.proj.bias, self.norm3.weight, self.norm3.bias)
            out["fold"] = {"a1": self.attn1.pack_folded(self.norm1.weight, self.norm1.bias),
                           "a2": self.attn2.pack_folded(self.norm2.weight, self.norm2.bias),
                           "ffw": wf[idx].contiguous(), "ffs": sf[idx].contiguous(), "ffc": cf[idx].contiguous()}
        return out

    def forward(self, x, context=None, B=1, stats=None, key_mass=None):
        """x: [B*N, C] bf16 tokens (reference _forward, attention.py:214-218).  stats: (table, partials per row) — the LayerNorm
        partial sums of x's rows written by the GEMM that produced x -> the three LayerNorms run inside the GEMM epilogues."""
        ops = _ops()
        p = self.packed()
        C = x.shape[1]
        edit = getattr(context, "edit", None)      # a prompt edit on this context also edits the block's self-attention
        if stats is not None and "fold" in p and (x.shape[0] // B) % 8 == 0 and x.shape[0] % 32 == 0:
            f = p["fold"]
            st1, parts1 = stats
            st2, st3 = ops.ln_stats_buffer(x.shape[0], C, x.device), ops.ln_stats_buffer(x.shape[0], C, x.device)
            x, parts2 = self.attn1.forward_folded(x, ops.LnFold(st1, parts1, C, self.norm1.eps), f["a1"], None, resid=x, B=B, stats_out=st2,
                                                 edit=edit, key_mass=key_mass)
            x, parts3 = self.attn2.forward_folded(x, ops.LnFold(st2, parts2, C, self.norm2.eps), f["a2"], context, resid=x, B=B, stats_out=st3)
            h = ops.gemm_ln(x, f["ffw"], bias=f["ffc"], act=ops.ACT_GEGLU, ln=ops.LnFold(st3, parts3, C, self.norm3.eps), colsum=f["ffs"])
            return ops.gemm(h, p["w2"], bias=p["b2"], resid=x)
        x = self.attn1(ops.layernorm(x, *p["norm1"], eps=self.norm1.eps), None, resid=x, B=B, edit=edit, key_mass=key_mass)
        x = self.attn2(ops.layernorm(x, *p["norm2"], eps=self.norm2.eps), context, resid=x, B=B)
        h = self.ff.net[0](ops.layernorm(x, *p["norm3"], eps=self.norm3.eps))
        return ops.gemm(h, p["w2"], bias=p["b2"], resid=x)


class SpatialTransformer(PackedModule):
    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0., context_dim=None, disable_self_attn=False):
        super().__init__()
        self.in_channels = in_channels
        inner_dim = n_heads * d_head
        self.norm = Normalize(in_channels)
        self.proj_in = nn.Conv2d(in_channels, inner_dim, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner_dim, n_heads, d_head, dropout=dropout, context_dim=context_dim,
                                   disable_self_attn=disable_self_attn) for _ in range(depth)])
        self.proj_out = zero_module(nn.Conv2d(inner_dim, in_channels, kernel_size=1, stride=1, padding=0))

    def _pack(self):
        return {"g": f32(self.norm.weight), "b": f32(self.norm.bias), "win": pack_conv1x1(self.proj_in.weight),
                "bin": f32(self.proj_in.bias), "wout": pack_conv1x1(self.proj_out.weight), "bout": f32(self.proj_out.bias)}

    def forward(self, x, context=None, ratio=1.0, acc=None, key_mass=None):
        """x: NHWC bf16 [B,H,W,C].  Returns ratio * proj_out(blocks(...)) + (acc if given else x):
        with acc=None, ratio=1 this is the reference forward (x + x_in, attention.py:255-266); with the
        running `acc` it is one term of VD_v2_0.context_mixing (vd.py:391-396) accumulated in the epilogue.
        key_mass: a KeyMass that the blocks' self-attention adds its key mass to (self-attention guidance)."""
        require_cuda(x, "SpatialTransformer")
        ops = _ops()
        p = self.packed()
        B, H, W, C = x.shape
        xn = ops.groupnorm(x, p["g"], p["b"], self.norm.eps)
        inner = p["win"].shape[0]
        if ln_fold_fits(inner, B, H, W):
            # proj_in also writes the LayerNorm statistics of its output rows: norm1 of the first block runs inside attn1's GEMMs
            st = ops.ln_stats_buffer(B * H * W, inner, x.device)
            t, parts = ops.gemm_ln(xn.view(B * H * W, C), p["win"], bias=p["bin"], stats_out=st)
            stats = (st, parts)
        else:
            stats = None
            t = ops.gemm(xn.view(B * H * W, C), p["win"], bias=p["bin"])
        for i, blk in enumerate(self.transformer_blocks):
            t = blk(t, context, B=B, stats=stats if i == 0 else None, key_mass=key_mass)
        base = x if acc is None else acc
        out = ops.gemm(t, p["wout"], bias=p["bout"], resid=base.view(B * H * W, -1), alpha=float(ratio))
        return out.view(B, H, W, -1)
