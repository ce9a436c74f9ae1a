"""VD_v2_0 — the multi-flow container of Versatile Diffusion on vdb200 kernels.
Reference: lib/model_zoo/vd.py:41-455.  Same constructor arguments, ModuleDicts (vae / ctx / diffuser),
schedule buffers, `to()` semantics and public methods that app.py and DDIMSampler use:
apply_model, apply_model_multicontext, context_mixing, vae_encode, vae_decode, ctx_encode, q_sample.
Training-only pieces (losses, EMA, logvar) are out of scope for the sampling hot path.
"""
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from lib.model_zoo.common.get_model import get_model, register
from lib.log_service import print_log
from .diffusion_utils import extract_into_tensor, make_beta_schedule, timestep_embedding, require_cuda
from .openaimodel import unet_walk

symbol = 'vd'


def _ops():
    from vdb200 import ops
    return ops


def highlight_print(info):
    print_log('')
    print_log(''.join(['#'] * (len(info) + 4)))
    print_log('# ' + info + ' #')
    print_log(''.join(['#'] * (len(info) + 4)))
    print_log('')


@register('vd_v2_0')
class VD_v2_0(nn.Module):
    def __init__(self, vae_cfg_list, ctx_cfg_list, diffuser_cfg_list, global_layer_ptr=None,
                 parameterization="eps", timesteps=1000, use_ema=False,
                 beta_schedule="linear", beta_linear_start=1e-4, beta_linear_end=2e-2, given_betas=None, cosine_s=8e-3,
                 loss_type="l2", l_simple_weight=1., l_elbo_weight=0., v_posterior=0., learn_logvar=False,
                 logvar_init=0, latent_scale_factor=None):
        super().__init__()
        assert parameterization in ["eps", "x0"], 'currently only supporting "eps" and "x0"'
        if use_ema:
            raise NotImplementedError("EMA is training-only (out of the sampling hot path)")
        self.parameterization = parameterization
        highlight_print("Running in {} mode".format(self.parameterization))
        self.vae = self.get_model_list(vae_cfg_list)
        self.ctx = self.get_model_list(ctx_cfg_list)
        self.diffuser = self.get_model_list(diffuser_cfg_list)
        self.global_layer_ptr = global_layer_ptr
        assert self.check_diffuser(), 'diffuser layers are not aligned!'
        self.use_ema = use_ema
        self.v_posterior = v_posterior
        self.device = 'cpu'
        self.register_schedule(given_betas=given_betas, beta_schedule=beta_schedule, timesteps=timesteps,
                               linear_start=beta_linear_start, linear_end=beta_linear_end, cosine_s=cosine_s)
        self.latent_scale_factor = {} if latent_scale_factor is None else dict(latent_scale_factor)
        self.parameter_group = {}
        for namei, diffuseri in self.diffuser.items():
            self.parameter_group.update({
                'diffuser_{}_{}'.format(namei, pgni): pgi for pgni, pgi in diffuseri.parameter_group.items()})

    def to(self, device):
        """Like the reference (vd.py:114-116): records .device and returns None."""
        self.device = device
        super().to(device)

    def get_model_list(self, cfg_list):
        net = nn.ModuleDict()
        for name, cfg in cfg_list:
            if isinstance(cfg, str):
                raise NotImplementedError("string-registered sub-models are not part of the hot path")
            net[name] = get_model()(cfg, verbose=False)
        return net

    def register_schedule(self, given_betas=None, beta_schedule="linear", timesteps=1000,
                          linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3):
        """fp64 numpy tables -> fp32 buffers, reference vd.py:127-185 (sampling-relevant subset + posterior)."""
        betas = given_betas if given_betas is not None else make_beta_schedule(
            beta_schedule, timesteps, linear_start=linear_start, linear_end=linear_end, cosine_s=cosine_s)
        alphas = 1. - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1., alphas_cumprod[:-1])
        timesteps, = betas.shape
        self.num_timesteps = int(timesteps)
        self.linear_start = linear_start
        self.linear_end = linear_end
        to_torch = partial(torch.tensor, dtype=torch.float32)
        self.register_buffer('betas', to_torch(betas))
        self.register_buffer('alphas_cumprod', to_torch(alphas_cumprod))
        self.register_buffer('alphas_cumprod_prev', to_torch(alphas_cumprod_prev))
        self.register_buffer('sqrt_alphas_cumprod', to_torch(np.sqrt(alphas_cumprod)))
        self.register_buffer('sqrt_one_minus_alphas_cumprod', to_torch(np.sqrt(1. - alphas_cumprod)))
        self.register_buffer('log_one_minus_alphas_cumprod', to_torch(np.log(1. - alphas_cumprod)))
        self.register_buffer('sqrt_recip_alphas_cumprod', to_torch(np.sqrt(1. / alphas_cumprod)))
        self.register_buffer('sqrt_recipm1_alphas_cumprod', to_torch(np.sqrt(1. / alphas_cumprod - 1)))
        posterior_variance = (1 - self.v_posterior) * betas * (1. - alphas_cumprod_prev) / (1. - alphas_cumprod) \
            + self.v_posterior * betas
        self.register_buffer('posterior_variance', to_torch(posterior_variance))
        self.register_buffer('posterior_log_variance_clipped', to_torch(np.log(np.maximum(posterior_variance, 1e-20))))
        self.register_buffer('posterior_mean_coef1', to_torch(betas * np.sqrt(alphas_cumprod_prev) / (1. - alphas_cumprod)))
        self.register_buffer('posterior_mean_coef2',
                             to_torch((1. - alphas_cumprod_prev) * np.sqrt(alphas) / (1. - alphas_cumprod)))

    def check_diffuser(self):
        order = None
        for diffuseri in self.diffuser.values():
            if order is None:
                order = diffuseri.layer_order
            elif order != diffuseri.layer_order:
                return False
        return True

    # ------------------------------------------------------------------ diffusion helpers
    def q_sample(self, x_start, t, noise=None):
        """sqrt(ac_t)*x0 + sqrt(1-ac_t)*noise (vd.py:221-224); per-row t -> one axpby launch per distinct row."""
        noise = torch.randn_like(x_start) if noise is None else noise
        require_cuda(x_start, "VD_v2_0.q_sample")
        ops = _ops()
        xs, nz = x_start.float().contiguous(), noise.float().contiguous()
        out = torch.empty_like(xs)
        a = self.sqrt_alphas_cumprod[t].tolist()
        b = self.sqrt_one_minus_alphas_cumprod[t].tolist()
        for i in range(xs.shape[0]):
            ops.axpby(xs[i], nz[i], a[i], b[i], out=out[i])
        return out.to(x_start.dtype)

    @torch.no_grad()
    def images_to_uint8(self, x):
        """Addition (SURVEY §8f rank 3): what app.py:319 does on the host with tvtrans.ToPILImage() — decoded images
        [n,3,H,W] in [0,1] -> uint8 [n,H,W,3] (x * 255 truncated), on the device: a quarter of the D2H bytes."""
        require_cuda(x, "VD_v2_0.images_to_uint8")
        return _ops().to_uint8_hwc(x.float().contiguous())

    @torch.no_grad()
    def vae_encode(self, x, which, **kwargs):
        scale = self.latent_scale_factor.get(which, None) if self.latent_scale_factor is not None else None
        if kwargs.get('out_posterior', False) or scale is None:
            return self.vae[which].encode(x, **kwargs)
        return self.vae[which].encode(x, post_scale=scale, **kwargs)   # scale * z fused into the sampling kernel

    @torch.no_grad()
    def vae_decode(self, z, which, **kwargs):
        scale = self.latent_scale_factor.get(which, None) if self.latent_scale_factor is not None else None
        return self.vae[which].decode(z, pre_scale=1.0 if scale is None else 1. / scale, **kwargs)

    @torch.no_grad()
    def ctx_encode(self, x, which, **kwargs):
        if which.find('vae_') == 0:
            return self.vae[which[4:]].encode(x, **kwargs)
        return self.ctx[which].encode(x, **kwargs)

    # ------------------------------------------------------------------ the UNet forward
    def time_source(self, x_type, multicontext):
        """Which diffuser owns time_embed: global_layer_ptr for apply_model (vd.py:339-342), diffuser[x_type]
        for apply_model_multicontext (vd.py:415-417)."""
        if multicontext or self.global_layer_ptr is None:
            return x_type
        return self.global_layer_ptr

    def eps_nhwc(self, x_nhwc, x_type, t_emb, c_types, contexts, ratios, time_from, key_mass=None):
        """Core of apply_model*: fp32 NHWC latent [B,H,W,4] + fp32 sinusoid [B,model_channels] -> fp32 NHWC eps.  key_mass: an
        attention.KeyMass that receives the mid block's self-attention key mass (lib/model_zoo/sag.py)."""
        table = self.diffuser[x_type].embed_table(t_emb, time_owner=self.diffuser[time_from])
        return unet_walk(self.diffuser[x_type], [self.diffuser[ct] for ct in c_types], x_nhwc, table, contexts, ratios, key_mass)

    def context_kv_signature(self, c_types, contexts):
        """Projects every context through the K / V^T weights of the cross-attention layers that will read it (a
        cache hit when the context is unchanged, an IN-PLACE refresh when a persistent context buffer was refilled)
        and returns the device addresses of those projections.  A captured DDIM-step graph reads exactly these
        buffers, so the sampler replays it only while the signature is unchanged."""
        from .attention import CrossAttention
        sig = []
        for ct, ctx in zip(c_types, contexts):
            for m in self.diffuser[ct].context_blocks.modules():
                if isinstance(m, CrossAttention) and not m.is_self:
                    k, vt = m.context_kv(ctx)[:2]
                    sig.append((k.data_ptr(), vt.data_ptr()))
        return tuple(sig)

    def _apply_model(self, x_type, x, timesteps, c_types, contexts, ratios, time_from):
        require_cuda(x, "VD_v2_0.apply_model")
        ops = _ops()
        t_emb = timestep_embedding(timesteps, self.diffuser[time_from].model_channels, repeat_only=False)
        if x.dim() == 2:
            # text latent [B, 768] (i2t / t2t flows, SURVEY §8f rank 4): the 0-D diffuser's data blocks take the flat latent
            if not getattr(self.diffuser[x_type], "dlayer_included", False):
                raise RuntimeError(f"diffuser['{x_type}'] was built without its data blocks: construct the model with the "
                                   "'openai_unet_0d_v1_dc' text diffuser (VDB_TEXT_FLOWS=1) for the text-latent flows")
            eps = self.eps_nhwc(x.float().contiguous(), x_type, t_emb, c_types, contexts, ratios, time_from)
            return eps.to(x.dtype)
        xh = ops.nchw_to_nhwc(x.float().contiguous())
        eps = self.eps_nhwc(xh, x_type, t_emb, c_types, contexts, ratios, time_from)
        return ops.nhwc_to_nchw(eps).to(x.dtype)

    def apply_model(self, x_info, timesteps, c_info):
        """vd.py:330-381: data blocks of diffuser[x_type], context blocks of diffuser[c_type]."""
        x_type, x = x_info['type'], x_info['x']
        c_type, c = c_info['type'], c_info['c']
        return self._apply_model(x_type, x, timesteps, [c_type], [c], [1.0], self.time_source(x_type, False))

    def context_mixing(self, x, emb, context_module_list, context_info_list, mixing_type):
        """vd.py:383-402 on NHWC bf16 activations ('attention' mixing; 'layer' picks one flow at random)."""
        context = [c_info['c'] for c_info in context_info_list]
        cratio = np.array([c_info['ratio'] for c_info in context_info_list], dtype=np.float64)
        cratio = cratio / cratio.sum()
        if mixing_type == 'attention':
            acc = None
            for module, c, r in zip(context_module_list, context, cratio):
                acc = module[0](x, c, ratio=float(r), acc=acc)
            return acc
        elif mixing_type == 'layer':
            ni = np.random.choice(len(context_module_list), p=cratio)
            return context_module_list[ni](x, emb, context[ni])
        raise ValueError(mixing_type)

    def apply_model_multicontext(self, x_info, timesteps, c_info_list, mixing_type='attention'):
        """vd.py:404-455: every 'c' slot = sum_i r_i * ST_i(h, c_i); time_embed of diffuser[x_type]."""
        if mixing_type != 'attention':
            raise NotImplementedError("only mixing_type='attention' is used by app.py")
        x_type, x = x_info['type'], x_info['x']
        return self._apply_model(x_type, x, timesteps, [ci['type'] for ci in c_info_list],
                                 [ci['c'] for ci in c_info_list], [ci['ratio'] for ci in c_info_list],
                                 self.time_source(x_type, True))
