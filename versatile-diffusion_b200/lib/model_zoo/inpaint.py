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


def check_inputs(x_info, shape):
    """The host-side refusals of a masked call -> (x0, mask).  Runs before any device work."""
    mask = x_info['inpaint_mask']
    if len(shape) != 4:
        raise ValueError(f"inpainting needs an image latent [bs, C, H, W], got shape {list(shape)} (a text latent?)")
    x0 = x_info.get('x0', None)
    if x0 is None:
        raise ValueError("inpaint_mask needs x_info['x0'], the latent of the image to keep")
    bs, C, H, W = shape
    if x0.dim() != 4 or x0.shape[0] not in (1, bs) or tuple(x0.shape[1:]) != (C, H, W):
        raise ValueError(f"x0: expected [{bs} or 1, {C}, {H}, {W}], got {tuple(x0.shape)}")
    mask_resolution(mask.shape, bs, H, W)
    if not bool(((mask >= 0) & (mask <= 1)).all()):
        raise ValueError("inpaint_mask: values must lie in [0, 1]")
    return x0, mask


def blend_table(alphas_prev):
    """fp32 [n, 2] rows {sqrt(a'), sqrt(1 - a')} in fp64 -> fp32, indexed by the grid index; row 0 is {1, 0}."""
    a = np.asarray(alphas_prev.cpu() if isinstance(alphas_prev, torch.Tensor) else alphas_prev, dtype=np.float64)
    t = np.stack([np.sqrt(a), np.sqrt(1.0 - a)], axis=1).astype(np.float32)
    t[0] = (1.0, 0.0)
    return t


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
