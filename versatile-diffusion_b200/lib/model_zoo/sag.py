"""Self-attention guidance (SAG) — guidance without a classifier from the UNet's own mid-block self-attention, inside the captured
DDIM / DPM-Solver++ step graph.

The reference has no SAG; this is an addition, and its semantics are specified here.  The method is Hong et al., "Improving Sample
Quality of Diffusion Models Using Self-Attention Guidance" (ICCV 2023), as diffusers' StableDiffusionSAGPipeline runs it: blur the
predicted clean image where the model attends most, re-noise it, run the UNet again, and push eps away from that degraded
prediction.  It needs no retraining.

API.  x_info['sag'] = sag.SelfAttentionGuidance(scale=0.75) on DDIMSampler.sample / sample_multicontext and DPMSolverSampler (same
methods).  scale must be finite and > 0; to turn SAG off, leave 'sag' out.  It combines with the img2img start ('x0'), 'xt',
'inpaint_mask', 'inversion' (with its mask) and eta > 0.  Notation: bs images, s the SAG scale, a_t = alphas_cumprod[t] at the step's
timestep t (the same for DDIM and DPM-Solver++).  Under CFG (guidance scale != 1) the UNet batch is [uncond ; cond].

1. Map.  The step's normal UNet pass also records the self-attention probabilities P[b, h, p, j] (softmax over keys j of
   scale q_p . k_j) of the mid block's SpatialTransformer (the 'c' of m_order), at N = hm * wm tokens: hm, wm are the latent sides
   halved with ceiling three times (8 x 8 at 512^2).  It records the rows SAG uses: the uncond rows [0, bs) under CFG, all (cond)
   rows without.  mass[b, j] = sum_i r_i (1/H) sum_h sum_p P_i[b, h, p, j] over the contexts i of the call with their normalised
   mixing ratios r_i (one context: r = 1).  The mask cell is M[b, j] = mass[b, j] > 1: the mean mass per key is exactly 1, so this
   marks the keys that get more than average attention.
2. Degrade.  e = e_u under CFG, e_c without.  x0 = (x_t - sqrt(1 - a_t) e) / sqrt(a_t).  blur is the depthwise 9 x 9 Gaussian of
   sigma 1 (1-D taps exp(-k^2 / 2), k = -4 .. 4, normalised to sum 1; the 2-D kernel their outer product) with reflect padding by 4
   (F.pad(mode='reflect')), so a latent side must be at least 5.  The mask is upsampled to the latent by nearest neighbour,
   src = floor(y hm / H) in integers.  x0_deg = M blur(x0) + (1 - M) x0 and x_deg = sqrt(a_t) x0_deg + sqrt(1 - a_t) e.
3. Second pass.  The UNet on x_deg (bs rows) at the same t with the uncond contexts (CFG) or the cond contexts: e_deg.  It reads
   items [0, bs) of the step's own context buffers, so the cached K / V^T of every cross-attention layer serve it unchanged.
4. Guide.  d = s (e - e_deg) is added to e_u and e_c in place, before the sampler's unchanged update:
   with CFG eps = e_u + g (e_c - e_u) + s (e_u - e_deg); without, eps = e_c + s (e_c - e_deg).

On the device: vdb_sattn_key_mass_f32 (inside the mid block's self-attention, two launches), vdb_sag_degrade_f32 and
vdb_sag_guide_f32; their per-step row {sqrt(a_t), sqrt(1 - a_t)} comes from a host-built table (fp64 -> fp32) read at the device
step counter, so one captured graph serves every step.  Each step runs 1.5 times the UNet items of an unguided step.

Refusals, before any device work.  NotImplementedError with 'windows' or 'regions' (they replace the UNet call) and with a
'prompt_edit' (its item tables index the CFG batch and know nothing of the second pass); on PLMSSampler and the single-step
p_sample_ddim(_multicontext).  ValueError for a text latent, a latent side below 5, a mid map of more than 4096 tokens, and an
x_info['sag'] that is not a SelfAttentionGuidance.  Without 'sag' nothing changes: the same launches, the same bits, the same graph
key.
"""
import math

import numpy as np
import torch

from .ddim import SamplerMode, buffers_key, refuse

MID_DOWNSAMPLES = 3     # the stride-2 convs before the mid block: channel_mult has four levels
MAX_MID_TOKENS = 4096


def _ops():
    from vdb200 import ops
    return ops


class SelfAttentionGuidance(object):
    """x_info['sag']: self-attention guidance at `scale` (finite, > 0)."""

    def __init__(self, scale=0.75):
        try:
            s = float(scale)
        except (TypeError, ValueError):
            raise ValueError(f"SelfAttentionGuidance: scale must be a real number, got {scale!r}") from None
        if not math.isfinite(s) or s <= 0:
            raise ValueError(f"SelfAttentionGuidance: scale must be finite and > 0 (to turn SAG off, omit it), got {scale!r}")
        self.scale = s


def mid_size(H, W):
    """The mid block's token grid (hm, wm) of an H x W latent: each stride-2 conv (kernel 3, padding 1) maps a side n to ceil(n / 2)."""
    for _ in range(MID_DOWNSAMPLES):
        H, W = (H + 1) // 2, (W + 1) // 2
    return H, W


def sag_table(alphas_cumprod, timesteps):
    """fp32 [len(timesteps), 2] rows {sqrt(a_t), sqrt(1 - a_t)} of a_t = alphas_cumprod[t] in fp64, indexed by the grid index."""
    a = np.asarray(alphas_cumprod.detach().cpu().numpy() if torch.is_tensor(alphas_cumprod) else alphas_cumprod,
                   dtype=np.float64)[np.asarray(timesteps)]
    return np.stack([np.sqrt(a), np.sqrt(1.0 - a)], axis=1).astype(np.float32)


class SelfAttention(SamplerMode):
    """x_info['sag'] in the sampler's walk: the step's eps from the recording pass, the degraded second pass and the guide."""

    def __init__(self, sampler, x_info, shape, c_infos):
        """The host-side refusals of a guided call, before any device work."""
        sag = x_info['sag']
        if not isinstance(sag, SelfAttentionGuidance):
            raise ValueError(f"x_info['sag'] must be a sag.SelfAttentionGuidance, got {type(sag).__name__}")
        refuse('sag', x_info, c_infos)
        if len(shape) != 4:
            raise ValueError(f"SAG needs an image latent [bs, C, H, W], got shape {list(shape)} (a text latent?)")
        H, W = shape[2], shape[3]
        if min(H, W) < 5:
            raise ValueError(f"SAG blurs with reflect padding by 4: latent sides must be >= 5, got {H} x {W}")
        self.hm, self.wm = mid_size(H, W)
        if self.hm * self.wm > MAX_MID_TOKENS:
            raise ValueError(f"SAG: the mid block's {self.hm} x {self.wm} tokens exceed {MAX_MID_TOKENS} (latent {H} x {W})")
        self.scale = sag.scale

    def prepare(self, sampler, run):
        """Refill the step table in place; the mass and the degraded latent are persistent buffers of the walk record."""
        st = run.walk
        if 'sag_tab' not in st:
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=run.device)
            st.update(sag_tab=z(1000, 2), sag_mass=z(run.bs, self.hm * self.wm), sag_x=z(run.bs, run.H, run.W, run.C))
        st['sag_tab'][:run.total].copy_(torch.from_numpy(sag_table(sampler.model.alphas_cumprod,
                                                                   sampler.ddim_timesteps[:run.total])))
        return ('sag', self.scale) + buffers_key(st['sag_tab'], st['sag_mass'], st['sag_x'])

    def eps(self, sampler, run):
        """zero the mass -> UNet pass 1 (recording) -> degrade -> UNet pass 2 on bs rows -> guide"""
        from .attention import KeyMass
        ops, w, bs, model = _ops(), run.walk, run.bs, sampler.model
        w['sag_mass'].zero_()
        t_emb = ops.timestep_embedding(w['ts'], run.mch, step_idx=w['idx'], batch=run.B)
        eps = model.eps_nhwc(w['x_in'], run.x_type, t_emb, run.c_types, run.ctxs, run.ratios, run.time_from,
                             key_mass=KeyMass(w['sag_mass']))
        e_u, e_c = (eps[:bs], eps[bs:]) if run.cfg else (None, eps)
        e_src = e_c if e_u is None else e_u
        ops.sag_degrade(run.x, e_src, w['sag_mass'], w['sag_tab'], w['idx'], self.hm, self.wm, out=w['sag_x'])
        e_deg = model.eps_nhwc(w['sag_x'], run.x_type, t_emb[:bs], run.c_types, run.ctxs, run.ratios, run.time_from)
        ops.sag_guide(e_u, e_c, e_deg, self.scale)
        return eps
