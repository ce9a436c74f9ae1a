"""Editing a real image — DDIM inversion and DiffEdit's automatic mask, inside the captured DDIM / DPM-Solver++ step graph.

The reference has no inversion and no editing; this is an addition, and its semantics are specified here.  Method: DDIM
inversion (the deterministic DDIM ODE run backwards from the image latent) and DiffEdit (Couairon et al., "DiffEdit:
Diffusion-based semantic image editing with mask guidance", ICLR 2023): the region to change is where the noise predictions
under the source and the target conditioning disagree; it is regenerated under the target, and outside it the walk replays the
inversion's trajectory.  The model needs no retraining.

Inversion.  DDIMSampler.invert(steps, x0, c_info, k=None) / invert_multicontext(steps, x0, c_info_list, k=None) -> Inversion.
  - x0: the image latent [bs or 1, 4, H, W], already scaled (net.vae_encode(img * 2 - 1, 'image')); bs is the contexts' batch.
  - The grid t_0 < ... < t_{n-1} is make_ddim_timesteps(steps); a_i = ddim_alphas[i], a'_i = ddim_alphas_prev[i].  Step i, for
    i = 0 ... k-1 (k defaults to n), with e the CFG-mixed eps at (x, t_i) under the inversion's contexts:
        x <- sqrt(a_i) (x - sqrt(1 - a'_i) e) / sqrt(a'_i) + sqrt(1 - a_i) e
    forward step i mirrored, with eps taken at the lower-noise point (the standard DDIM-inversion approximation).  It is
    vdb_ddim_cfg_step with the row {a'_i, a_i, 0, sqrt(1 - a'_i)} (inversion_rows: fp64 -> fp32); the step counter counts up.
  - Trajectory: fp32 NHWC [k+1, bs, H, W, C]; slot 0 is x0, slot i+1 the latent after step i, at level a_i, which is exactly
    where forward step i starts.  vdb_latent_store_slot_f32 writes slot idx + 1 from inside the captured step graph.
  - The walk runs on the sampler's step graph (the first step eager, then replays), in its own persistent state, so a cached
    graph replays on a new image and does not evict the sampling graph.  DDIM only: DPMSolverSampler.invert and
    PLMSSampler.invert raise NotImplementedError; a text latent [n, 768] and contexts of different batches raise ValueError.

Sampling from an inversion.  x_info = {'type': 'image', 'inversion': inv[, 'inpaint_mask': m]} on DDIMSampler.sample /
sample_multicontext and DPMSolverSampler (same methods; its targets are DDIM's a'_i).
  - The walk starts at slot k and visits grid points k-1 ... 0.  A steps or latent shape other than the inversion's raises
    ValueError, and so do 'xt', 'x0' or 'x0_forward_timesteps' given with 'inversion'.
  - m: 1 = regenerate, 0 = keep, [bs or 1, 1, H, W] or [bs or 1, 1, 8H, 8W], values in [0, 1] (as for inpainting).  After forward
    step i, per element in fp32 with the formula and op order of vdb_inpaint_blend_f32:
        x <- m x + (1 - m) slot_i
    (vdb_inversion_blend_f32, one launch in the step graph; under CFG it also writes the duplicate half).  The kept value is the
    trajectory, never re-noised x0, and no noise is drawn.  Slot 0 is x0, so the kept region of the result is x0 bit for bit.
  - Without 'inversion' nothing changes: the same launches, the same bits, the same graph key.

Mask (diffedit_mask(net, x0, src, tgt, steps=50, strength=0.5, n_draws=10, ratio=3.0, grid='uniform'), the paper's rule as
diffusers' StableDiffusionDiffEditPipeline.generate_mask applies it).  src / tgt: a context dict, or a list of them (multi-context);
every context of both sides has the batch bs (ValueError otherwise, before any device work).
  - k = int(steps * strength), t_m = t_{k-1} on the time grid `grid` (edit passes the sampler's): the level of slot k, where
    edit's walk starts.  D = n_draws draws
    x_d = sqrt(ac[t_m]) x0 + sqrt(1 - ac[t_m]) z_d, z_d from torch.randn (torch.manual_seed fixes the mask).
  - E_src, E_tgt: the CFG-mixed eps of each side at its own scale; one UNet call per side on a batch of D * bs (doubled under
    CFG), draw d of image b at row d * bs + b.
  - Per image: d(p) = 1/(D C) sum_d sum_c |E_tgt - E_src|, mu = mean_p d(p), cap = ratio mu,
    mask(p) = min(d(p), cap) / cap >= 0.5 ? 1 : 0 (all 0 when cap == 0).  vdb_diffedit_mask_f32: one CTA per image, sums in
    an order fixed by the shape, so the mask is bit-reproducible.  -> fp32 [bs, 1, H, W], ready for 'inpaint_mask'.

edit(net, sampler, image, src, tgt, steps=50, strength=0.5, mask='auto', n_draws=10): encode image ([n, 3, 8H, 8W] in [0, 1]),
invert under src at scale 1 to k = int(steps * strength), build the mask ('auto': diffedit_mask; a tensor: as given; None: no mask,
pure inversion-anchored regeneration), sample under tgt (a list: multi-context, e.g. VD's text + image edit), decode.
-> (images [n, 3, 8H, 8W] in [0, 1], mask or None).  No paste-back: inpaint.composite does that.
"""
import numpy as np
import torch

from .ddim import SamplerMode, buffers_key, refuse
from .diffusion_utils import make_ddim_timesteps, to_numpy


def _ops():
    from vdb200 import ops
    return ops


class Inversion(object):
    """A DDIM inversion: the trajectory (fp32 NHWC [k+1, bs, H, W, C], slot 0 = x0) and what a sampling call must match."""

    def __init__(self, trajectory, steps, k, timesteps, shape):
        self.trajectory = trajectory
        self.steps, self.k = int(steps), int(k)
        self.timesteps = np.asarray(timesteps)
        self.shape = tuple(shape)                # [bs, C, H, W] of the latent
        self.bs = self.shape[0]
        self.xt = _ops().nhwc_to_nchw(trajectory[k].contiguous())   # slot k, NCHW: where the walk starts

    def __repr__(self):
        return f"Inversion(steps={self.steps}, k={self.k}, shape={list(self.shape)})"


def inversion_rows(alphas, alphas_prev, k):
    """fp32 [k, 4] rows {a'_i, a_i, 0, sqrt(1 - a'_i)} of inversion steps 0 ... k-1, built in fp64."""
    a, ap = to_numpy(alphas, np.float64)[:k], to_numpy(alphas_prev, np.float64)[:k]
    return np.stack([ap, a, np.zeros_like(a), np.sqrt(1.0 - ap)], axis=1).astype(np.float32)


def check_invert_inputs(x0, bs, k, n):
    """The host-side refusals of an inversion -> k.  Runs before any device work."""
    if x0.dim() != 4:
        raise ValueError(f"inversion needs an image latent [bs, C, H, W], got shape {list(x0.shape)} (a text latent?)")
    if x0.shape[0] not in (1, bs):
        raise ValueError(f"x0: expected a batch of {bs} or 1 (the contexts' batch), got {tuple(x0.shape)}")
    k = n if k is None else int(k)
    if not 1 <= k <= n:
        raise ValueError(f"k = {k}: need 1 <= k <= {n}, the grid points of the walk")
    return k


class FromInversion(SamplerMode):
    """x_info['inversion'] in the sampler's walk: the start at slot k, and with an inpaint_mask the trajectory blend after every
    step."""

    def __init__(self, sampler, x_info, shape, c_infos):
        """The host-side refusals of a sampling call from an inversion, before any device work."""
        inv = self.inv = x_info['inversion']
        if not isinstance(inv, Inversion):
            raise ValueError(f"x_info['inversion']: expected an Inversion (DDIMSampler.invert), got {type(inv).__name__}")
        refuse('inversion', x_info, c_infos)
        if not np.array_equal(np.asarray(sampler.ddim_timesteps), inv.timesteps):
            raise ValueError(f"the inversion was made with steps={inv.steps}: sample with the same steps")
        if tuple(shape) != inv.shape:
            raise ValueError(f"shape {list(shape)} differs from the inversion's {list(inv.shape)}")
        self.mask = x_info.get('inpaint_mask', None)
        if self.mask is not None:
            from .inpaint import check_mask
            check_mask(self.mask, *inv.shape[:1], *inv.shape[2:])

    def start(self, sampler, x_info, shape, dtype, device):
        return self.inv.xt.to(dtype).to(device), sampler.ddim_timesteps[:self.inv.k]

    def prepare(self, sampler, run):
        if self.mask is None:
            return ()
        from .inpaint import load_mask
        inv = self.inv
        st = run.walk
        if 'traj' not in st or st['traj'].shape[0] < inv.k or st['traj'].shape[1:] != inv.trajectory.shape[1:]:
            st['traj'] = torch.zeros((max(inv.k, len(sampler.ddim_timesteps)),) + tuple(inv.trajectory.shape[1:]),
                                     dtype=torch.float32, device=run.device)
        if 'mask' not in st:
            st['mask'] = torch.zeros(run.bs, run.H * run.W, dtype=torch.float32, device=run.device)
        st['traj'][:inv.k].copy_(inv.trajectory[:inv.k])
        self.traj, self.mask_rows = st['traj'], load_mask(st['mask'], self.mask, run.W)
        return ('inversion',) + buffers_key(self.traj, self.mask_rows)

    def after_update(self, run):
        if self.mask is not None:
            _ops().inversion_blend(run.x, self.traj, self.mask_rows, run.walk['idx'], x_dup=run.x_dup)


def context_batch(c_infos, scale):
    """The batch that every context of c_infos has -> bs.  ValueError when a conditioning (or, under CFG, an
    unconditional_conditioning) has another: the UNet would read one context row per latent row past its end."""
    bs = c_infos[0]['conditioning'].shape[0]
    keys = ('conditioning', 'unconditional_conditioning') if scale != 1. else ('conditioning',)
    for i, ci in enumerate(c_infos):
        for key in keys:
            if ci[key].shape[0] != bs:
                raise ValueError(f"context {i}: '{key}' has a batch of {ci[key].shape[0]}, expected {bs} (all contexts must "
                                 f"share one batch)")
    return bs


def _side(c):
    """A side's contexts -> (c_infos, multi, scale, bs), checked on the host."""
    c_infos = list(c) if isinstance(c, (list, tuple)) else [c]
    scale = float(c_infos[0]['unconditional_guidance_scale'])
    for ci in c_infos:
        if float(ci['unconditional_guidance_scale']) != scale:
            raise ValueError("A different unconditional guidance scale between different context is not allowed!")
    return c_infos, isinstance(c, (list, tuple)), scale, context_batch(c_infos, scale)


def _side_contexts(c_infos, scale, D, device):
    """CFG-doubled context tensors of a side, repeated over the D draws."""
    ctxs = []
    for ci in c_infos:
        cc = ci['conditioning'].to(device).repeat(D, 1, 1)
        ctxs.append(torch.cat([ci['unconditional_conditioning'].to(device).repeat(D, 1, 1), cc]) if scale != 1. else cc)
    return ctxs


@torch.no_grad()
def diffedit_mask(net, x0, src, tgt, steps=50, strength=0.5, n_draws=10, ratio=3.0, grid='uniform'):
    """DiffEdit's {0, 1} latent mask [bs, 1, H, W] (1 = edit) from the disagreement of the src and tgt noise predictions, at the
    level of slot k of the inversion over `grid` (the sampler's time grid)."""
    ts = make_ddim_timesteps(grid, steps, net.num_timesteps, verbose=False, alphas_cumprod=net.alphas_cumprod)
    n = len(ts)
    k = int(steps * strength)
    if not 1 <= k <= n:
        raise ValueError(f"strength {strength} at {steps} steps gives k = {k}: need 1 <= k <= {n}")
    D = int(n_draws)
    if D < 1:
        raise ValueError(f"n_draws must be >= 1, got {n_draws}")
    if not ratio > 0:
        raise ValueError(f"ratio must be > 0, got {ratio}")
    if x0.dim() != 4:
        raise ValueError(f"diffedit_mask needs an image latent [bs, C, H, W], got shape {list(x0.shape)}")
    sides = [_side(src), _side(tgt)]
    bs = sides[0][3]
    if sides[1][3] != bs:
        raise ValueError(f"tgt's contexts have a batch of {sides[1][3]}, src's {bs}: both sides must share one batch")
    if x0.shape[0] not in (1, bs):
        raise ValueError(f"x0: expected a batch of {bs} or 1 (the contexts' batch), got {tuple(x0.shape)}")
    ops = _ops()
    device = torch.device(net.device)
    _, C, H, W = x0.shape
    t_m = int(ts[k - 1])
    ac = float(net.alphas_cumprod[t_m])
    z = torch.randn(D * bs, C, H, W)                      # torch's CPU generator: torch.manual_seed fixes the mask
    x0r = x0.to(device=device, dtype=torch.float32).expand(bs, C, H, W).repeat(D, 1, 1, 1).contiguous()
    xd = ops.nchw_to_nhwc(ops.axpby(x0r, z.to(device), np.sqrt(ac), np.sqrt(1.0 - ac)))
    eps = []
    for c_infos, multi, scale, _ in sides:
        ctxs = _side_contexts(c_infos, scale, D, device)
        cfg = scale != 1.
        x_in = torch.cat([xd, xd]) if cfg else xd
        time_from = net.time_source('image', multi)
        t_emb = ops.timestep_embedding(torch.full((x_in.shape[0],), t_m, dtype=torch.int64, device=device),
                                       net.diffuser[time_from].model_channels)
        e = net.eps_nhwc(x_in, 'image', t_emb, [ci['type'] for ci in c_infos], ctxs,
                         [float(ci.get('ratio', 1.0)) for ci in c_infos], time_from)
        eps.append(((e[:D * bs], e[D * bs:]) if cfg else (None, e), scale))
    (su, sc), s_src = eps[0]
    (tu, tc), s_tgt = eps[1]
    m = ops.diffedit_mask(su, sc, s_src, tu, tc, s_tgt, D, ratio)
    return m.view(bs, 1, H, W)


@torch.no_grad()
def edit(net, sampler, image, src, tgt, steps=50, strength=0.5, mask='auto', n_draws=10):
    """Edit image ([n, 3, 8H, 8W] in [0, 1]) from the src conditioning to the tgt conditioning -> (images in [0, 1], mask).
    mask: 'auto' (diffedit_mask), a latent or pixel mask tensor (1 = edit), or None (no mask)."""
    n, _, H8, W8 = image.shape
    k = int(steps * strength)
    x0 = net.vae_encode(image * 2 - 1, 'image')
    src_l = list(src) if isinstance(src, (list, tuple)) else [src]
    inv_src = [dict(ci, unconditional_guidance_scale=1.0) for ci in src_l]
    if len(inv_src) > 1:
        inv = sampler.invert_multicontext(steps, x0, inv_src, k=k)
    else:
        inv = sampler.invert(steps, x0, inv_src[0], k=k)
    if isinstance(mask, str):
        if mask != 'auto':
            raise ValueError(f"mask: 'auto', a tensor or None, got {mask!r}")
        mask = diffedit_mask(net, x0, src, tgt, steps=steps, strength=strength, n_draws=n_draws, grid=sampler.grid)
    x_info = {'type': 'image', 'inversion': inv}
    if mask is not None:
        x_info['inpaint_mask'] = mask
    shape = [n, 4, H8 // 8, W8 // 8]
    if isinstance(tgt, (list, tuple)):
        z, _ = sampler.sample_multicontext(steps=steps, shape=shape, x_info=x_info, c_info_list=list(tgt), verbose=False)
    else:
        z, _ = sampler.sample(steps=steps, shape=shape, x_info=x_info, c_info=tgt, verbose=False)
    return net.vae_decode(z, 'image'), mask
