"""Schedules, sinusoidal embedding and module helpers of the sampling path
(reference lib/model_zoo/diffusion_utils.py:8-59, 79-82, 131-151, 175-209, 235-240)."""
import math

import numpy as np
import torch
import torch.nn as nn


def make_beta_schedule(schedule, n_timestep, linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3):
    """fp64 beta tables (reference :8-30); always built on the host, even under a torch.device(cuda) context."""
    cpu = torch.device("cpu")
    if schedule == "linear":
        betas = torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64, device=cpu) ** 2
    elif schedule == "cosine":
        ts = torch.arange(n_timestep + 1, dtype=torch.float64, device=cpu) / n_timestep + cosine_s
        alphas = torch.cos(ts / (1 + cosine_s) * np.pi / 2).pow(2)
        alphas = alphas / alphas[0]
        betas = np.clip(1 - alphas[1:] / alphas[:-1], a_min=0, a_max=0.999)
    elif schedule == "sqrt_linear":
        betas = torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64, device=cpu)
    elif schedule == "sqrt":
        betas = torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64, device=cpu) ** 0.5
    else:
        raise ValueError(f"schedule '{schedule}' unknown.")
    return betas.numpy() if isinstance(betas, torch.Tensor) else np.asarray(betas)


GRIDS = ("uniform", "trailing", "karras")     # the samplers' `grid` option


def make_ddim_timesteps(ddim_discr_method, num_ddim_timesteps, num_ddpm_timesteps, verbose=True, alphas_cumprod=None):
    """Ascending integer timesteps of the walk (T = num_ddpm_timesteps, S = num_ddim_timesteps); step i goes from t_i to
    t_{i-1}, step 0 to ac[0].
      - uniform (reference :32-46): range(0, T, T // S) + 1.  The walk starts below T - 1: at 951 for 20 steps.
      - quad (reference): linspace(0, sqrt(0.8 T), S)^2 + 1.
      - trailing (diffusers' timestep_spacing="trailing"): round(arange(T, 0, -T / S)) - 1, S points, so the walk starts at T - 1.
      - karras (Karras et al. 2022, rho = 7): S sigmas from sigma(T - 1) down to sigma(1), sigma(t) = sqrt((1 - ac[t]) / ac[t])
        in fp64 from the fp32 alphas_cumprod (so it needs them), evenly spaced in sigma^(1/7); each is mapped to t by linear
        interpolation of t over log sigma(t) (diffusers' _sigma_to_t), rounded to the nearest integer, repeats dropped.  The
        grid ends at t = 1 as uniform does, so step 0 never has a zero step.  Where the low sigmas lie closer than one timestep
        the grid has fewer than S points and the walk takes fewer steps: 98 at S = 100 on the linear schedule."""
    if ddim_discr_method == "uniform":
        c = num_ddpm_timesteps // num_ddim_timesteps
        steps_out = np.asarray(list(range(0, num_ddpm_timesteps, c))) + 1
    elif ddim_discr_method == "quad":
        steps_out = ((np.linspace(0, np.sqrt(num_ddpm_timesteps * .8), num_ddim_timesteps)) ** 2).astype(int) + 1
    elif ddim_discr_method == "trailing":
        # np.arange's length is computed in floating point and is S + 1 for some S (61, 103, ...), the extra point at about 0:
        # the grid is its first S points
        ts = np.round(np.arange(num_ddpm_timesteps, 0, -num_ddpm_timesteps / num_ddim_timesteps))[:num_ddim_timesteps]
        steps_out = np.sort(ts.astype(np.int64) - 1)
    elif ddim_discr_method == "karras":
        if num_ddim_timesteps < 2:
            raise ValueError(f"the karras grid needs at least 2 steps, got {num_ddim_timesteps}")
        if alphas_cumprod is None:
            raise ValueError("the karras grid needs the model's alphas_cumprod")
        ac = to_numpy(alphas_cumprod, np.float32).astype(np.float64)
        sigma = np.sqrt((1.0 - ac) / ac)
        lo, hi = sigma[1] ** (1 / 7), sigma[num_ddpm_timesteps - 1] ** (1 / 7)
        j = np.arange(num_ddim_timesteps, dtype=np.float64) / (num_ddim_timesteps - 1)
        t = np.interp(np.log((hi + j * (lo - hi)) ** 7), np.log(sigma), np.arange(num_ddpm_timesteps, dtype=np.float64))
        steps_out = np.unique(np.rint(t).astype(np.int64))
    else:
        raise NotImplementedError(f'There is no ddim discretization method called "{ddim_discr_method}"')
    if verbose:
        print(f"Selected timesteps for ddim sampler: {steps_out}")
    return steps_out


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta, verbose=True):
    """reference :48-59 (same mixed tensor/ndarray dtype walk: alphas keeps alphacums' type)."""
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    if verbose:
        print(f"Selected alphas for ddim sampler: a_t: {alphas}; a_(t-1): {alphas_prev}")
        print(f"For the chosen value of eta, which is {eta}, this results in the following sigma_t schedule "
              f"for ddim sampler {sigmas}")
    return sigmas, alphas, alphas_prev


def to_numpy(x, dtype=None):
    """A tensor on any device, or anything np.asarray takes -> ndarray (of dtype when given)."""
    return np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=dtype)


def extract_into_tensor(a, t, x_shape):
    b, *_ = t.shape
    out = a.gather(-1, t)
    return out.reshape(b, *((1,) * (len(x_shape) - 1)))


def timestep_embedding(timesteps, dim, max_period=10000, repeat_only=False):
    """[cos | sin] sinusoid (reference :131-151) on the vdb200 kernel; CPU tensors raise (no CPU path in the product)."""
    if repeat_only:
        return timesteps[:, None].expand(-1, dim)
    require_cuda(timesteps, "timestep_embedding")
    from vdb200 import ops
    return ops.timestep_embedding(timesteps.long().contiguous(), dim, max_period)


def noise_like(x, repeat=False):
    noise = torch.randn_like(x)
    if repeat:
        noise = noise[0:1].repeat(x.shape[0], *((1,) * (len(x.shape) - 1)))
    return noise


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


class GroupNorm32(nn.GroupNorm):
    """Parameter holder with the reference's key names (weight, bias); eps 1e-5 (reference :175-191).
    The arithmetic runs in vdb200's groupnorm kernel from the owning block."""


def normalization(channels):
    return GroupNorm32(32, channels)


def conv_nd(dims, *args, **kwargs):
    if dims != 2:
        raise ValueError("the H100 hot path is 2-D only")
    return nn.Conv2d(*args, **kwargs)


def linear(*args, **kwargs):
    return nn.Linear(*args, **kwargs)


# ------------------------------------------------------------------------------------------------
# packing support shared by every kernel-backed module
# ------------------------------------------------------------------------------------------------
_pack_epoch = [0]


def pack_epoch():
    """Bumped whenever any module drops its kernel-layout weights (.to / .half / load_state_dict / explicit
    invalidate_packed): captured CUDA graphs hold pointers to the packed copies, so samplers key their graphs on it."""
    return _pack_epoch[0]


class PackedMixin(object):
    """Lazily repacked kernel-side weights for an nn.Module.

    Parameters keep the reference's names/shapes/dtypes (the checkpoint ABI); `packed()` builds the
    bf16/fp32 kernel-layout copies on first use and is invalidated by .to()/.half()/.cuda() and by
    load_state_dict (in-place edits of .data are not tracked: call invalidate_packed())."""
    _packed = None

    def _apply(self, fn, *a, **k):
        self.invalidate_packed()
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self.invalidate_packed()
        return super()._load_from_state_dict(*a, **k)

    def invalidate_packed(self):
        self._packed = None
        _pack_epoch[0] += 1

    def packed(self):
        if self._packed is None:
            with torch.no_grad():
                self._packed = self._pack()
        return self._packed

    def _pack(self):
        raise NotImplementedError


class PackedModule(PackedMixin, nn.Module):
    pass


def require_cuda(t, who):
    if not t.is_cuda:
        raise RuntimeError(f"{who}: the H100 build has no CPU path — move the model and inputs to a CUDA device "
                           "(the CPU reference lives in oracle/, for tests only)")


def bf16(t):
    return t.detach().to(torch.bfloat16).contiguous()


def f32(t):
    return t.detach().to(torch.float32).contiguous()


def pack_conv3x3(w):
    """[Cout, Cin, 3, 3] -> bf16 [Cout, (ky, kx, ci)]"""
    return bf16(w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1))


def fold_upsample_conv3x3(w):
    """Weights of "nearest-2x upsample, then 3x3 conv (pad 1)" folded onto the SOURCE image.

    Output pixel (2y+py, 2x+px) reads upsampled rows 2y+py+ky-1, ky in {0,1,2}, i.e. source rows y + floor((py+ky-1)/2):
    parity 0 -> {y-1 (ky 0), y (ky 1, 2)}, parity 1 -> {y (ky 0, 1), y+1 (ky 2)}; the same along x.  Tap (ty, tx) of
    parity (py, px) therefore reads source pixel (y + ty - 1 + py, x + tx - 1 + px) with the SUM of the 3x3 weights that land
    on it (summed in fp32, rounded to bf16 once).  The zero padding of the upsampled image coincides with the zero padding
    of the source, so the result is exact up to that rounding.
    w [Cout, Cin, 3, 3] -> bf16 [4 (py*2+px), Cout, 4*Cin] with K ordered (ty, tx, ci) — conv modes 3..6 of vdb_conv3x3_bf16."""
    w = w.detach().float()
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}     # parity -> (3x3 taps folded into tap 0, into tap 1)
    out = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for ty in (0, 1):
                for tx in (0, 1):
                    acc = 0
                    for ky in groups[py][ty]:
                        for kx in groups[px][tx]:
                            acc = acc + w[:, :, ky, kx]
                    taps.append(acc)                                # [Cout, Cin]
            out.append(torch.stack(taps, dim=1).reshape(w.shape[0], -1))   # [Cout, (ty,tx,ci)]
    return torch.stack(out).to(torch.bfloat16).contiguous()


UPSAMPLE_FOLD_MIN_PIXELS = 2048


def upsample_fold_enabled(n_source_pixels, n_out):
    """Nearest-2x upsample folded into the following 3x3 conv (+1.1 % on the C2 bench): fold when the source grid is large
    enough to fill the machine without split-K (the four parity convs each see only B*H*W output pixels) and the conv's
    n_out output channels suit the interleaved TMA-store epilogue (n_out % 32 == 0)."""
    return n_source_pixels >= UPSAMPLE_FOLD_MIN_PIXELS and n_out % 32 == 0


def pack_conv1x1(w):
    return bf16(w.detach().reshape(w.shape[0], -1))
