"""Inpainting — keep a region of an image and regenerate the rest, inside the captured DDIM / DPM-Solver++ step graph.

The reference has no inpainting; this is an addition, and its semantics are specified here.  The method is blended latent
diffusion, the `mask` / `x0` arguments of CompVis latent-diffusion's DDIMSampler: after every step the region to keep is
overwritten with the original latent re-noised to the step's noise level.  The model needs no retraining.

API.  x_info = {'type': 'image', 'x0': x0, 'inpaint_mask': m[, 'x0_forward_timesteps': k]} on DDIMSampler.sample /
sample_multicontext and DPMSolverSampler (same methods), with any context set-up (single, dual, multi).
  - x0: the image latent [bs or 1, 4, H, W], already scaled (net.vae_encode(img, 'image')).
  - m: 1 marks what to generate, 0 what to keep (the convention of painted masks; LDM's `mask` is the opposite).  Shape
    [bs or 1, 1, H, W] at latent resolution or [bs or 1, 1, 8H, 8W] at pixel resolution; values in [0, 1], so the mask may be
    soft.  A pixel mask becomes a latent mask by the max over each 8x8 cell (latent_mask, vdb_mask_to_latent): any latent cell
    that touches a generated pixel is regenerated.

Blend after step i.  Step i goes from grid index i to its target point, of cumulative alpha a' (DDIM's ddim_alphas_prev[i];
DPM-Solver++ uses the same targets).  In fp32 per element, with z_i a fresh standard normal per element and step:
    x' <- m x' + (1 - m) (sqrt(a') x0 + sqrt(1 - a') z_i)
The rows {sqrt(a'), sqrt(1 - a')} are a host-built table (blend_table, fp64 -> fp32) indexed by the device step counter; the last
step (i = 0) uses the row {1, 0}, so the kept region of the returned latent is exactly x0.  m = 1 and m = 0 select exactly, so a
hard mask leaves the generated region as the step wrote it.  The blend runs after the step's update and before the counter moves,
on the eager and the graph path alike, so eta > 0 and DPM-Solver++ inherit it; under CFG it also writes the duplicate half.

Start.  With x0_forward_timesteps = k: the img2img start, unchanged (all of x0 noised to t_k, then the first k grid points).
Without it: the full walk from x_T (x_info['xt'], else torch.randn as without a mask), whose kept region is set once to
sqrt(ac[t_top]) x0 + sqrt(1 - ac[t_top]) x_T, reusing x_T's own draw.

Noise.  Philox4x32-10 at counter (element quad, step index i, "inpt", 0) under a 64-bit key; each counter gives four normals by
two Box-Muller pairs with u = (b + 0.5) 2^-32.  The key is drawn from torch's CPU generator at the start of each call, so
torch.manual_seed fixes the result; it is drawn only when a mask is given, so unmasked runs consume the generator as before.

Paste-back.  composite(decoded, image, pixel_mask) = m decoded + (1 - m) image per pixel after the VAE decode: optional, for a
user who prefers the original pixels outside the mask to the VAE's reconstruction of them.

Refusals.  ValueError for a text latent ([n, 768]), for an x0 or mask whose shape matches neither resolution or batch, for mask
values outside [0, 1], and for an inpaint_mask without x0.  PLMSSampler raises NotImplementedError.  Without inpaint_mask
nothing changes: the same launches, the same bits, the same graph key.
"""
import numpy as np
import torch

from .ddim import SamplerMode, buffers_key
from .diffusion_utils import to_numpy


def _ops():
    from vdb200 import ops
    return ops


def mask_resolution(mask_shape, bs, H, W):
    """'latent' for [bs or 1, 1, H, W], 'pixel' for [bs or 1, 1, 8H, 8W]; ValueError otherwise."""
    s = tuple(mask_shape)
    if len(s) == 4 and s[0] in (1, bs) and s[1] == 1:
        if s[2:] == (H, W):
            return 'latent'
        if s[2:] == (8 * H, 8 * W):
            return 'pixel'
    raise ValueError(f"inpaint_mask: expected [{bs} or 1, 1, {H}, {W}] (latent) or [{bs} or 1, 1, {8 * H}, {8 * W}] (pixel), "
                     f"got {s}")


def check_mask(mask, bs, H, W):
    """The refusals of an inpaint_mask (also the mask of a walk from an inversion, lib/model_zoo/edit.py)."""
    mask_resolution(mask.shape, bs, H, W)
    if not bool(((mask >= 0) & (mask <= 1)).all()):
        raise ValueError("inpaint_mask: values must lie in [0, 1]")


def blend_table(alphas_prev):
    """fp32 [n, 2] rows {sqrt(a'), sqrt(1 - a')} in fp64 -> fp32, indexed by the grid index; row 0 is {1, 0}."""
    a = to_numpy(alphas_prev, np.float64)
    t = np.stack([np.sqrt(a), np.sqrt(1.0 - a)], axis=1).astype(np.float32)
    t[0] = (1.0, 0.0)
    return t


def load_mask(dst, mask, W):
    """Copy a latent or pixel mask [n, 1, ., .] into rows 0 .. n-1 of the device buffer dst [bs, H * W] -> the rows a blend
    reads: dst, or dst[:1] for one mask shared by every item."""
    mask = mask.to(device=dst.device, dtype=torch.float32).contiguous()
    if mask.shape[-1] != W:
        mask = _ops().mask_to_latent(mask)
    dst[:mask.shape[0]].copy_(mask.view(mask.shape[0], dst.shape[1]))
    return dst if mask.shape[0] != 1 else dst[:1]


class Inpainting(SamplerMode):
    """x_info['inpaint_mask'] in the sampler's walk: the start of a full walk, and the blend after every step."""

    def __init__(self, sampler, x_info, shape, c_infos):
        """The host-side refusals of a masked call, before any device work."""
        self.mask = x_info['inpaint_mask']
        if len(shape) != 4:
            raise ValueError(f"inpainting needs an image latent [bs, C, H, W], got shape {list(shape)} (a text latent?)")
        self.x0 = x_info.get('x0', None)
        if self.x0 is None:
            raise ValueError("inpaint_mask needs x_info['x0'], the latent of the image to keep")
        bs, C, H, W = shape
        if self.x0.dim() != 4 or self.x0.shape[0] not in (1, bs) or tuple(self.x0.shape[1:]) != (C, H, W):
            raise ValueError(f"x0: expected [{bs} or 1, {C}, {H}, {W}], got {tuple(self.x0.shape)}")
        check_mask(self.mask, bs, H, W)
        self.full_walk = x_info.get('x0_forward_timesteps', None) is None
        # the Philox key, from torch's CPU generator; drawn only when a mask is given, after every refusal
        self.seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)

    def start(self, sampler, x_info, shape, dtype, device):
        if self.full_walk:      # a masked full walk starts from x_T as an unmasked one does, never from the img2img start
            self.x_T, ts = sampler._initial_latent(shape, {k: v for k, v in x_info.items() if k != 'x0'}, dtype, device)
            return self.x_T, ts
        # the img2img start noises x0 row by row: a batch-1 x0 is noised once per item
        return sampler._initial_latent(shape, dict(x_info, x0=self.x0.expand(shape[0], *self.x0.shape[1:])), dtype, device)

    def prepare(self, sampler, run):
        """With x_T (the full walk) the kept region of the latent becomes x0 noised to t_top with x_T's own draw."""
        ops = _ops()
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=run.device)
        st = run.walk
        if 'x0' not in st:
            st.update(x0=z(run.bs, run.H, run.W, run.C), mask=z(run.bs, run.H * run.W), blend=z(1000, 2),
                      seed=z(1, dtype=torch.int64))
        st['x0'].copy_(ops.nchw_to_nhwc(self.x0.to(device=run.device, dtype=torch.float32).contiguous()))   # broadcasts [1]
        self.mask_rows = load_mask(st['mask'], self.mask, run.W)
        st['blend'][:run.total].copy_(torch.from_numpy(blend_table(sampler.ddim_alphas_prev[:run.total])))
        st['seed'].copy_(self.seed)
        if self.full_walk:
            a_top = float(sampler.ddim_alphas[run.total - 1])
            row = torch.tensor([[np.sqrt(a_top), np.sqrt(1.0 - a_top)]], dtype=torch.float32, device=run.device)
            ops.inpaint_blend(run.x, st['x0'], self.mask_rows, row, torch.zeros(1, dtype=torch.int32, device=run.device),
                              noise=ops.nchw_to_nhwc(self.x_T.float().contiguous()))
        return ('inpaint',) + buffers_key(st['x0'], self.mask_rows, st['blend'], st['seed'])

    def after_update(self, run):
        w = run.walk
        _ops().inpaint_blend(run.x, w['x0'], self.mask_rows, w['blend'], w['idx'], seed=w['seed'], x_dup=run.x_dup)


def latent_mask(pixel_mask):
    """Pixel mask [n, 1, 8H, 8W] -> latent mask [n, 1, H, W]: the max over each 8x8 cell."""
    return _ops().mask_to_latent(pixel_mask.float().contiguous())


def composite(decoded, image, pixel_mask):
    """m decoded + (1 - m) image per pixel: decoded / image [n, C, 8H, 8W], pixel_mask [n or 1, 1, 8H, 8W]."""
    return _ops().composite(decoded.float().contiguous(), image.float().contiguous(), pixel_mask.float().contiguous())


@torch.no_grad()
def inpaint(net, sampler, image, mask, c_info, steps, x0_forward_timesteps=None, paste_back=True, **kw):
    """Encode image ([n, 3, 8H, 8W] in [0, 1], as ToTensor gives it and vae_decode returns it), sample with the pixel mask
    ([n or 1, 1, 8H, 8W], 1 = generate), decode, and paste the kept pixels back unless paste_back is False.  c_info: one
    context dict, or a list for sample_multicontext."""
    n, _, H8, W8 = image.shape
    x_info = {'type': 'image', 'x0': net.vae_encode(image * 2 - 1, 'image'), 'inpaint_mask': mask}
    if x0_forward_timesteps is not None:
        x_info['x0_forward_timesteps'] = x0_forward_timesteps
    shape = [n, 4, H8 // 8, W8 // 8]
    kw.setdefault('verbose', False)
    if isinstance(c_info, (list, tuple)):
        z, _ = sampler.sample_multicontext(steps=steps, shape=shape, x_info=x_info, c_info_list=list(c_info), **kw)
    else:
        z, _ = sampler.sample(steps=steps, shape=shape, x_info=x_info, c_info=c_info, **kw)
    out = net.vae_decode(z, 'image')
    return composite(out, image, mask.to(out.device)) if paste_back else out
