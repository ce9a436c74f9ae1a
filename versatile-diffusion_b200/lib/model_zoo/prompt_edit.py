"""Prompt-to-Prompt editing (Hertz et al., "Prompt-to-Prompt Image Editing with Cross Attention Control", ICLR 2023) inside the
captured step graph of DDIMSampler and DPMSolverSampler.  The reference has no prompt editing, so this docstring is the
specification.

Usage: row 0 of the batch is the source prompt, rows 1 .. n-1 are targets; c_info['prompt_edit'] = replace(...) / refine(...) /
reweight(...) / PromptEdit(...) on the text context that carries the edit.  With several contexts (sample_multicontext) the edit
acts only on that context; the others keep their own attention.

Notation: n prompts, L = 77 key positions, T = the walk's step count, i = 0 .. T-1 the position in the walk (0 is the noisiest
step).  Positions relate to the sampler's device counter by idx = T-1-i.

Start.  Without 'xt', x_T is one torch.randn([1, C, H, W]) draw expanded to all n rows, as P2P runs every prompt from the same
noise.  'xt' may be [1 or n, C, H, W].  ValueError before any device work: 'x0', 'inpaint_mask' or 'inversion' together with
'prompt_edit'; a text latent; a non-text context carrying the edit; a conditioning batch other than n.  PLMSSampler and the
single-step p_sample_ddim(_multicontext) refuse the edit with NotImplementedError.

Per target b, host-side, fp64 then fp32: an L x L matrix A_b and an L-vector beta_b, with c_b the equalizer (1 where no weight
is given):
  replace:  A = M diag(c), beta = 0, M the word-swap mapper.
  refine:   A[k, j] = [map(j) = k] alpha_j c_j, beta = (1 - alpha) * c, map and alpha from the token alignment.
  reweight: A = diag(c), beta = 0, usually with the target prompt equal to the source.

Edited contexts.  ctx'_b = A_b ctx_b and ctx''_b = diag(beta_b) ctx_b, from the target's fp32 conditioning (the product in
fp64), rounded to bf16 in a persistent context buffer [uncond rows; cond rows; ctx'_1 ..; ctx''_1 .. (refine only)].  Their
K / V^T come from CrossAttention.context_kv like any other context: projected once per call, outside the graph.

Cross-attention (every attn2 of the edited context).  The conditional row of target b, at walk positions i < floor(cross_steps T):
  O = softmax(s q_src K(ctx_src)^T) V(ctx'_b)  [+ softmax(s q_b K(ctx_b)^T) V(ctx''_b) when beta_b != 0].
At other positions it is the row's own attention.  Unconditional rows and the source row are never edited, as in P2P, which
edits only the conditional half.  VD's to_v has no bias, so in exact arithmetic this equals P2P's edit on the probabilities:
(attn_src M) * c, or (alpha * attn_src[:, map] + (1 - alpha) * attn_tgt) * c.  One indexed flash-attention launch
(vdb_attention_bf16 with an items table) does it; the refinement's second term is a second launch that accumulates into the output.

Self-attention (attn1 of the edited context's SpatialTransformers).  Only at layers whose token grid is at most (H/4)(W/4)
tokens (H/4 and W/4 rounded up as the UNet's stride-2 convolutions round them); that is P2P's 16^2 limit at 512^2.  At
positions i < floor(self_steps T), the conditional row of target b becomes softmax(s q_src k_src^T) V_b.

Word maps.  Blend words give a 0/1 weight table w [n, L].  The map map[b, p] is zeroed at the start of the walk.  In every step,
each cross-attention layer at 1/4 of the latent side (at full size: two on the way down, three on the way up; the 1/8 mid block
is not included) adds sum_h sum_j w[b, j] softmax(s q_b K(ctx_b)^T)[h, p, j] to it, for every conditional row b
(vdb_xattn_word_map_f32).  These are the row's own pre-edit probabilities.  P2P's code records them after its in-place edit;
here they are recorded before it.

Local blend.  It runs after the step's update, at positions i >= floor(blend_start T) (vdb_local_blend_f32):
  pooled_b = 3x3 max-pool (stride 1, pad 1) of map[b];
  up_b = nearest upsampling to H x W, where latent pixel y reads map row floor(y h / H);
  mask_b = up_b / max(pooled_b) > threshold (false when the max is 0), and m_b = mask_b or mask_0;
  for b >= 1: x_b <- m_b ? x_b : x_0, a selection, so that outside the mask x_b takes x_0's bits.  The CFG duplicate half is
  written too.
Defaults: threshold = 0.3, blend_start = 0, cross_steps = 0.8, self_steps = 0.4.

Builders.  replace, refine and reweight run on the host.  They take any tokenizer with encode(str) -> ids (start and end tokens
included, as CLIPTokenizer returns) and decode([id]) -> str; on an installation, the CLIP tokenizer the text encoder loads.
  A word (prompts split on spaces) owns the token positions its pieces take, counted from 1.
  replace needs equal word counts.  A swapped word with s source and t target tokens maps one-to-one if s = t.  Otherwise every
  source token of the word maps to every target token of the word with weight 1/t.  Other positions map in order, shifted by
  the accumulated length difference, while both are < L.  Any target position left over maps to itself.
  refine globally aligns the two token sequences: match +1, mismatch -1, gap -1.  On ties the traceback prefers the diagonal,
  then a target insertion.  A target token aligned to a source token (match or mismatch) gets alpha = 1 and map(j) = that
  token; an inserted token gets alpha = 0.  Positions past the target sequence map to themselves with alpha = 1.
  reweight(words, values) sets c on the tokens of those words.
  The low-level PromptEdit(A, beta, cross_steps, self_steps, blend=None, threshold=0.3, blend_start=0.0) takes the tables
  directly.

Without 'prompt_edit' nothing changes: the same launches, the same bits and the same graph key.

Not covered: P2P's per-word time windows (one window per edit here), null-text inversion, edits of image contexts, and
combinations with inpainting or an inversion blend.
"""
import math

import numpy as np
import torch

from .ddim import SamplerMode, buffers_key, refuse

L_MAX = 77


def _ops():
    from vdb200 import ops
    return ops


# ---------------------------------------------------------------------------------------------------- tokens and words
def word_positions(tok, text):
    """Token positions (counted from 1, after the start token) of each space-separated word of text."""
    out, pos = [], 1
    for word in text.split(' '):
        k = len(tok.encode(word)) - 2
        out.append(list(range(pos, pos + k)))
        pos += k
    return out


def positions_of(tok, text, words):
    """Token positions of the given words (strings, matched against every occurrence, or word indices) in text."""
    if isinstance(words, (str, int)):
        words = [words]
    split, wp = text.split(' '), word_positions(tok, text)
    out = []
    for w in words:
        idx = [w] if isinstance(w, int) else [i for i, s in enumerate(split) if s == w]
        if not idx:
            raise ValueError(f"word {w!r} is not in the prompt {text!r}")
        for i in idx:
            out += wp[i]
    return out


def replacement_mapper(tok, src, tgt, L=L_MAX):
    """The word-swap mapper M [L, L] (fp64): M[k, j] is the weight of source position k in target position j."""
    ws, wt = src.split(' '), tgt.split(' ')
    if len(ws) != len(wt):
        raise ValueError(f"replace needs prompts of equal word counts: {len(ws)} and {len(wt)} words")
    ps, pt = word_positions(tok, src), word_positions(tok, tgt)
    swaps = [(ps[w], pt[w]) for w in range(len(ws)) if ws[w] != wt[w]]
    M = np.zeros((L, L))
    i = j = cur = 0
    while i < L and j < L:
        if cur < len(swaps) and swaps[cur][0] and swaps[cur][0][0] == i:
            s, t = swaps[cur]
            if len(s) == len(t):
                for a, b in zip(s, t):
                    if a < L and b < L:
                        M[a, b] = 1.0
            else:
                for a in s:
                    for b in t:
                        if a < L and b < L:
                            M[a, b] = 1.0 / len(t)
            cur += 1
            i += len(s)
            j += len(t)
        else:
            M[i, j] = 1.0
            i += 1
            j += 1
    while j < L:            # target positions left over when the source ran out first
        M[j, j] = 1.0
        j += 1
    return M


def align(x, y):
    """Global alignment of token sequences x (source) and y (target): match +1, mismatch -1, gap -1; on ties the traceback
    prefers the diagonal, then a target insertion.  -> for each target token, the aligned source index or -1 (inserted)."""
    nx, ny = len(x), len(y)
    S = np.zeros((nx + 1, ny + 1))
    S[:, 0] = -np.arange(nx + 1)
    S[0, :] = -np.arange(ny + 1)
    for i in range(1, nx + 1):
        for j in range(1, ny + 1):
            S[i, j] = max(S[i - 1, j - 1] + (1 if x[i - 1] == y[j - 1] else -1), S[i, j - 1] - 1, S[i - 1, j] - 1)
    out = [-1] * ny
    i, j = nx, ny
    while i > 0 or j > 0:
        if i > 0 and j > 0 and S[i, j] == S[i - 1, j - 1] + (1 if x[i - 1] == y[j - 1] else -1):
            out[j - 1] = i - 1
            i, j = i - 1, j - 1
        elif j > 0 and S[i, j] == S[i, j - 1] - 1:
            j -= 1                                  # target insertion: out[j] stays -1
        else:
            i -= 1                                  # source deletion
    return out


def refinement_map(tok, src, tgt, L=L_MAX):
    """(map [L] int, alpha [L] fp64) of the token alignment; positions past the target sequence map to themselves."""
    x, y = list(tok.encode(src)), list(tok.encode(tgt))
    a = align(x, y)
    mp, alpha = np.arange(L), np.ones(L)
    for j in range(min(len(y), L)):
        if a[j] < 0:
            mp[j], alpha[j] = j, 0.0
        else:
            mp[j] = a[j]
    return mp, alpha


def equalizer(tok, text, words=None, values=None, L=L_MAX):
    """c [L] fp64: 1, and values on the tokens of words (a number or one per word)."""
    c = np.ones(L)
    if words is None:
        return c
    words = [words] if isinstance(words, (str, int)) else list(words)
    values = [values] * len(words) if np.isscalar(values) else list(values)
    if len(values) != len(words):
        raise ValueError(f"reweight: {len(words)} words and {len(values)} values")
    for w, v in zip(words, values):
        for p in positions_of(tok, text, w):
            if p < L:
                c[p] = float(v)
    return c


def blend_table(tok, prompts, blend_words, L=L_MAX):
    """w [n, L] fp32: 1 on the tokens of each prompt's blend words."""
    if len(blend_words) != len(prompts):
        raise ValueError(f"blend_words: one list per prompt ({len(prompts)}), got {len(blend_words)}")
    w = np.zeros((len(prompts), L), np.float32)
    for b, (p, ws) in enumerate(zip(prompts, blend_words)):
        for q in positions_of(tok, p, ws):
            if q < L:
                w[b, q] = 1.0
    return w


# ---------------------------------------------------------------------------------------------------- the edit
class PromptEdit(object):
    """The edit's tables: A [n-1, L, L] and beta [n-1, L] per target (stored fp32), the windows, and the optional local blend
    (w [n, L] word weights, threshold, blend_start)."""

    def __init__(self, A, beta, cross_steps=0.8, self_steps=0.4, blend=None, threshold=0.3, blend_start=0.0):
        A = np.asarray(A, dtype=np.float64)
        beta = np.asarray(beta, dtype=np.float64)
        if A.ndim != 3 or A.shape[1] != A.shape[2] or A.shape[0] < 1:
            raise ValueError(f"A: expected [n-1, L, L] with n >= 2, got {A.shape}")
        if beta.shape != A.shape[:2]:
            raise ValueError(f"beta: expected {A.shape[:2]}, got {beta.shape}")
        for name, v in (("cross_steps", cross_steps), ("self_steps", self_steps), ("blend_start", blend_start)):
            if not 0.0 <= float(v) <= 1.0:
                raise ValueError(f"{name} must lie in [0, 1], got {v}")
        if not math.isfinite(float(threshold)):
            raise ValueError(f"threshold must be finite, got {threshold}")
        self.A, self.beta = A.astype(np.float32), beta.astype(np.float32)
        self.n, self.L = A.shape[0] + 1, A.shape[1]
        self.cross_steps, self.self_steps = float(cross_steps), float(self_steps)
        self.blend = None if blend is None else np.asarray(blend, dtype=np.float32)
        if self.blend is not None and self.blend.shape != (self.n, self.L):
            raise ValueError(f"blend: expected [{self.n}, {self.L}], got {self.blend.shape}")
        self.threshold, self.blend_start = float(threshold), float(blend_start)
        self.has_beta = bool(np.any(self.beta != 0))

    def edited_contexts(self, cond):
        """[ctx'_1 ..; ctx''_1 .. (when some beta != 0)] fp32 [(n-1)(1 or 2), L, C] from the fp32 conditioning [n, L, C]."""
        c = cond.detach().to(device='cpu', dtype=torch.float64)
        A, beta = torch.from_numpy(self.A).double(), torch.from_numpy(self.beta).double()
        out = [A @ c[1:]]
        if self.has_beta:
            out.append(beta[:, :, None] * c[1:])
        return torch.cat(out).float()

    def tables(self, T, cfg):
        """Host tables of a walk of T steps, indexed by the device counter idx = T-1-i -> dict of int32 arrays:
        'cross' / 'self' [T, 3, B] {bq, bk, bv} per output item, 'cross2' [T, 3, B] (bv = -1: skip) when some beta != 0, and
        'flags' [T] of the local blend.  B = 2n with CFG (rows [uncond; cond]), else n; the edited contexts follow at B."""
        n = self.n
        B = 2 * n if cfg else n
        c0 = n if cfg else 0
        ident = np.broadcast_to(np.arange(B, dtype=np.int32), (T, 3, B)).copy()
        cross, selfm = ident.copy(), ident.copy()
        cross2 = np.full((T, 3, B), -1, np.int32) if self.has_beta else None
        tc, ts = int(math.floor(self.cross_steps * T)), int(math.floor(self.self_steps * T))
        tb = int(math.floor(self.blend_start * T))
        flags = np.zeros(T, np.int32)
        for i in range(T):
            idx = T - 1 - i
            for t in range(1, n):
                r = c0 + t
                if i < tc:
                    cross[idx, :, r] = (c0, c0, B + t - 1)
                    if cross2 is not None and np.any(self.beta[t - 1] != 0):
                        cross2[idx, :, r] = (r, r, B + n - 1 + t - 1)
                if i < ts:
                    selfm[idx, :, r] = (c0, c0, r)
            flags[idx] = int(self.blend is not None and i >= tb)
        return {'cross': cross, 'self': selfm, 'cross2': cross2, 'flags': flags}


def _prompts_tok(tok, prompts):
    if len(prompts) < 2:
        raise ValueError("a prompt edit needs a source and at least one target prompt")
    return [len(tok.encode(p)) for p in prompts]


def _weights(tok, prompts, equalize):
    """c [n-1, L] of the targets from equalize = None or (words, values)."""
    return np.stack([equalizer(tok, p, *(equalize or (None, None))) for p in prompts[1:]])


def _blend(tok, prompts, blend_words):
    return None if blend_words is None else blend_table(tok, prompts, blend_words)


def replace(tok, prompts, cross_steps=0.8, self_steps=0.4, blend_words=None, equalize=None, threshold=0.3, blend_start=0.0):
    """Word swap: A_b = M_b diag(c_b), beta = 0.  equalize: optional (words, values) weights on the targets' tokens."""
    _prompts_tok(tok, prompts)
    c = _weights(tok, prompts, equalize)
    A = np.stack([replacement_mapper(tok, prompts[0], p) * c[b][None, :] for b, p in enumerate(prompts[1:])])
    return PromptEdit(A, np.zeros(A.shape[:2]), cross_steps, self_steps, _blend(tok, prompts, blend_words), threshold, blend_start)


def refine(tok, prompts, cross_steps=0.8, self_steps=0.4, blend_words=None, equalize=None, threshold=0.3, blend_start=0.0):
    """Added or changed words: A[k, j] = [map(j) = k] alpha_j c_j, beta = (1 - alpha) c from the token alignment."""
    _prompts_tok(tok, prompts)
    c = _weights(tok, prompts, equalize)
    A, beta = [], []
    for b, p in enumerate(prompts[1:]):
        mp, alpha = refinement_map(tok, prompts[0], p)
        a = np.zeros((L_MAX, L_MAX))
        a[mp, np.arange(L_MAX)] = alpha * c[b]
        A.append(a)
        beta.append((1.0 - alpha) * c[b])
    return PromptEdit(np.stack(A), np.stack(beta), cross_steps, self_steps, _blend(tok, prompts, blend_words), threshold,
                      blend_start)


def reweight(tok, prompts, words, values, cross_steps=0.8, self_steps=0.4, blend_words=None, threshold=0.3, blend_start=0.0):
    """Attention reweighting: A_b = diag(c_b) with c on the tokens of words in target b, beta = 0."""
    _prompts_tok(tok, prompts)
    c = _weights(tok, prompts, (words, values))
    A = np.stack([np.diag(cb) for cb in c])
    return PromptEdit(A, np.zeros(A.shape[:2]), cross_steps, self_steps, _blend(tok, prompts, blend_words), threshold, blend_start)


# ---------------------------------------------------------------------------------------------------- sampler side
def quarter(side):
    """The token side of the UNet level at 1/4 of the latent side (two stride-2 convolutions, each rounding up)."""
    return ((side + 1) // 2 + 1) // 2


class EditState(object):
    """What the attention layers of the edited context read during a walk (carried on its PaddedContext as `edit`): the device
    item tables, the step counter, the word weights and maps.  The sampler keeps it and refills it in place."""

    def __init__(self, n, cfg, ctx_batch, has_beta, blend, h4, w4, device):
        self.args = (n, cfg, ctx_batch, has_beta, blend, h4, w4)
        self.n, self.c0, self.B = n, (n if cfg else 0), (2 * n if cfg else n)
        self.ctx_batch, self.has_beta, self.blend, self.h4, self.w4 = ctx_batch, has_beta, blend, h4, w4
        z = lambda *s: torch.zeros(*s, dtype=torch.int32, device=device)
        self.cross, self.selfm, self.flags = z(1000, 3, self.B), z(1000, 3, self.B), z(1000)
        self.cross2 = z(1000, 3, self.B) if has_beta else None
        self.w = torch.zeros(n, L_MAX, dtype=torch.float32, device=device) if blend else None
        self.map = torch.zeros(n, h4 * w4, dtype=torch.float32, device=device) if blend else None
        self.idx, self.threshold = None, 0.3

    def fill(self, ed, T, cfg, idx):
        tabs = ed.tables(T, cfg)
        for name, dst in (('cross', self.cross), ('self', self.selfm), ('cross2', self.cross2), ('flags', self.flags)):
            if dst is not None:
                dst[:T].copy_(torch.from_numpy(tabs[name]))
        if self.blend:
            self.w.copy_(torch.from_numpy(ed.blend))
            self.map.zero_()
        self.idx, self.threshold = idx, ed.threshold

    # read by CrossAttention
    def items(self, cross, N):
        if cross:
            return self.cross
        return self.selfm if N <= self.h4 * self.w4 else None

    def maps_at(self, N):
        return self.blend and N == self.h4 * self.w4


class PromptEditing(SamplerMode):
    """A context's 'prompt_edit' in the sampler's walk: one start noise for every prompt, the edited context with its EditState,
    and the local blend after every step."""

    def __init__(self, sampler, x_info, shape, c_infos):
        """Refuse what the edit does not support, before any device work."""
        carriers = [i for i, ci in enumerate(c_infos) if ci.get('prompt_edit', None) is not None]
        if len(carriers) != 1:
            raise ValueError(f"one context may carry 'prompt_edit', got {len(carriers)}")
        i = self.i = carriers[0]
        ed = self.ed = c_infos[i]['prompt_edit']
        if not isinstance(ed, PromptEdit):
            raise ValueError(f"'prompt_edit' must be a PromptEdit, got {type(ed).__name__}")
        refuse('prompt_edit', x_info, c_infos)
        if len(shape) != 4 or x_info.get('type', 'image') != 'image':
            raise ValueError("'prompt_edit' edits image latents [n, C, H, W]; a text latent cannot be edited")
        if c_infos[i].get('type') != 'text':
            raise ValueError(f"'prompt_edit' must ride on a text context, got {c_infos[i].get('type')!r}")
        for ci in c_infos:
            for k in ('conditioning', 'unconditional_conditioning'):
                if ci.get(k, None) is not None and ci[k].shape[0] != ed.n:
                    raise ValueError(f"'prompt_edit' of {ed.n} prompts needs a {k} batch of {ed.n}, got {ci[k].shape[0]}")
        if c_infos[i]['conditioning'].shape[1] != ed.L:
            raise ValueError(f"'prompt_edit' tables of {ed.L} positions, the context has {c_infos[i]['conditioning'].shape[1]}")
        if shape[0] != ed.n:
            raise ValueError(f"'prompt_edit' of {ed.n} prompts needs a batch of {ed.n}, got {shape[0]}")
        xt = x_info.get('xt', None)
        if xt is not None and (xt.dim() != 4 or xt.shape[0] not in (1, ed.n) or tuple(xt.shape[1:]) != tuple(shape[1:])):
            raise ValueError(f"'xt' must be [1 or {ed.n}, {', '.join(map(str, shape[1:]))}], got {tuple(xt.shape)}")

    def start(self, sampler, x_info, shape, dtype, device):
        """every prompt starts from the same noise: one draw, or the given x_T, expanded to the n rows"""
        xt = x_info.get('xt', None)
        if xt is None:
            xt = torch.randn([1] + list(shape[1:]), device=device, dtype=dtype)
        return sampler._initial_latent(shape, dict(x_info, xt=xt.expand(list(shape))), dtype, device)

    def prepare(self, sampler, run):
        """Swap the edited context for its persistent extended buffer [context rows; edited contexts], which carries the
        EditState, and refill that state in place."""
        from .attention import PaddedContext
        ed, i, cfg = self.ed, self.i, run.cfg
        c = run.c_infos[i]['c']
        ext = torch.cat([c.float(), ed.edited_contexts(run.c_infos[i]['conditioning']).to(c.device)])
        buf = sampler._ctx_buffer(('prompt_edit', i), ext)
        es = run.walk.get('prompt_edit')
        args = (ed.n, cfg, ext.shape[0], ed.has_beta, ed.blend is not None, quarter(run.H), quarter(run.W))
        if es is None or es.args != args:
            es = run.walk['prompt_edit'] = EditState(*args, run.device)
        es.fill(ed, run.total, cfg, run.walk['idx'])
        run.ctxs[i] = PaddedContext(buf, c.shape[1], edit=es)
        self.es = es
        return ('prompt_edit', ed.n, ed.has_beta, es.blend, es.threshold) + buffers_key(es.cross, es.selfm, es.cross2, es.flags,
                                                                                         es.w, es.map)

    def after_update(self, run):
        es = self.es
        if es.blend:
            _ops().local_blend(run.x, es.map, es.flags, run.walk['idx'], es.h4, es.w4, es.threshold, x_dup=run.x_dup)
