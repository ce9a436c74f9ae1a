"""DDIMSampler on vdb200 kernels — same public surface as the reference (lib/model_zoo/ddim.py:10-298):
make_schedule, sample, ddim_sampling, p_sample_ddim and the *_multicontext twins.

Fast path (eta == 0, no noise dropout): the whole DDIM step — sinusoid, time MLP, all ResBlock emb
projections, the 46-block UNet walk over the CFG-doubled batch, and the fused CFG + x_{t-1} update —
is captured ONCE as a CUDA graph whose per-step scalars (timestep, a_t, a_prev, sigma, sqrt(1-a_t))
live in device tables indexed by a device-side step counter; the 50-step loop is 50 graph replays with
no host<->device traffic (the reference does ~15 tiny kernels + 4 H2D fills per step, ddim.py:159-171).
The latent stays fp32 NHWC between steps; NCHW conversion happens only at the API boundary.
"""
import numpy as np
import torch

from .diffusion_utils import make_ddim_sampling_parameters, make_ddim_timesteps, noise_like, require_cuda


def _ops():
    from vdb200 import ops
    return ops


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        super().__init__()
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.use_cuda_graph = kwargs.get("use_cuda_graph", True)
        self._graphs = {}
        self._inv_graphs = {}

    def register_buffer(self, name, attr):
        # the reference forces .to('cuda') here (ddim.py:17-21); follow the model's device instead
        if isinstance(attr, torch.Tensor) and str(self.model.device) != 'cpu' and attr.device != torch.device(self.model.device):
            attr = attr.to(torch.device(self.model.device))
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=True):
        """reference ddim.py:23-56 (same fp64/fp32 dtype walk)."""
        self.ddim_timesteps = make_ddim_timesteps(ddim_discr_method=ddim_discretize, num_ddim_timesteps=ddim_num_steps,
                                                  num_ddpm_timesteps=self.ddpm_num_timesteps, verbose=verbose)
        alphas_cumprod = self.model.alphas_cumprod
        assert alphas_cumprod.shape[0] == self.ddpm_num_timesteps, 'alphas have to be defined for each timestep'
        to_torch = lambda x: x.clone().detach().to(torch.float32).to(self.model.device)
        self.register_buffer('betas', to_torch(self.model.betas))
        self.register_buffer('alphas_cumprod', to_torch(alphas_cumprod))
        self.register_buffer('alphas_cumprod_prev', to_torch(self.model.alphas_cumprod_prev))
        ac = alphas_cumprod.cpu()
        self.register_buffer('sqrt_alphas_cumprod', to_torch(np.sqrt(ac)))
        self.register_buffer('sqrt_one_minus_alphas_cumprod', to_torch(np.sqrt(1. - ac)))
        self.register_buffer('log_one_minus_alphas_cumprod', to_torch(np.log(1. - ac)))
        self.register_buffer('sqrt_recip_alphas_cumprod', to_torch(np.sqrt(1. / ac)))
        self.register_buffer('sqrt_recipm1_alphas_cumprod', to_torch(np.sqrt(1. / ac - 1)))
        ddim_sigmas, ddim_alphas, ddim_alphas_prev = make_ddim_sampling_parameters(
            alphacums=ac, ddim_timesteps=self.ddim_timesteps, eta=ddim_eta, verbose=verbose)
        self.register_buffer('ddim_sigmas', ddim_sigmas)
        self.register_buffer('ddim_alphas', ddim_alphas)
        self.register_buffer('ddim_alphas_prev', ddim_alphas_prev)
        self.register_buffer('ddim_sqrt_one_minus_alphas', np.sqrt(1. - ddim_alphas))
        sigmas_for_original_sampling_steps = ddim_eta * torch.sqrt(
            (1 - self.alphas_cumprod_prev) / (1 - self.alphas_cumprod) * (1 - self.alphas_cumprod / self.alphas_cumprod_prev))
        self.register_buffer('ddim_sigmas_for_original_num_steps', sigmas_for_original_sampling_steps)

    # ------------------------------------------------------------------ reference-shaped entry points
    @torch.no_grad()
    def sample(self, steps, shape, x_info, c_info, eta=0., temperature=1., noise_dropout=0., verbose=True,
               log_every_t=100):
        self.make_schedule(ddim_num_steps=steps, ddim_eta=eta, verbose=verbose)
        if verbose:
            print(f'Data shape for DDIM sampling is {shape}, eta {eta}')
        return self.ddim_sampling(shape, x_info=x_info, c_info=c_info, noise_dropout=noise_dropout,
                                  temperature=temperature, log_every_t=log_every_t)

    @torch.no_grad()
    def sample_multicontext(self, steps, shape, x_info, c_info_list, eta=0., temperature=1., noise_dropout=0.,
                            verbose=True, log_every_t=100):
        self.make_schedule(ddim_num_steps=steps, ddim_eta=eta, verbose=verbose)
        if verbose:
            print(f'Data shape for DDIM sampling is {shape}, eta {eta}')
        return self.ddim_sampling_multicontext(shape, x_info=x_info, c_info_list=c_info_list,
                                               noise_dropout=noise_dropout, temperature=temperature,
                                               log_every_t=log_every_t)

    @torch.no_grad()
    def ddim_sampling(self, shape, x_info, c_info, noise_dropout=0., temperature=1., log_every_t=100):
        return self._run(shape, x_info, [c_info], False, noise_dropout, temperature, log_every_t)

    @torch.no_grad()
    def ddim_sampling_multicontext(self, shape, x_info, c_info_list, noise_dropout=0., temperature=1.,
                                   log_every_t=100):
        scale = c_info_list[0]['unconditional_guidance_scale']
        for ci in c_info_list:
            assert scale == ci['unconditional_guidance_scale'], \
                "A different unconditional guidance scale between different context is not allowed!"
        return self._run(shape, x_info, c_info_list, True, noise_dropout, temperature, log_every_t)

    # ------------------------------------------------------------------ the loop
    def _initial_latent(self, shape, x_info, dtype, device):
        """ddim.py:94-105: injected x_T ('xt'), img2img start (x0 + q_sample) or fresh noise; or slot k of an inversion and the
        first k grid points (lib/model_zoo/edit.py)."""
        timesteps = self.ddim_timesteps
        if x_info.get('inversion', None) is not None:
            inv = x_info['inversion']
            x, timesteps = inv.xt.to(dtype).to(device), timesteps[:inv.k]
        elif x_info.get('xt', None) is not None:
            x = x_info['xt'].to(dtype).to(device)       # (the reference's `.astype` here is a bug, ddim.py:95)
        elif x_info.get('x0', None) is not None:
            x0 = x_info['x0'].type(dtype).to(device)
            ts = np.repeat(timesteps[x_info['x0_forward_timesteps']], shape[0])
            ts = torch.Tensor(ts).long().to(device)
            timesteps = timesteps[:x_info['x0_forward_timesteps']]
            x = self.model.q_sample(x0, ts)
        else:
            x = torch.randn(shape, device=device, dtype=dtype)
        return x, timesteps

    def _run(self, shape, x_info, c_infos, multi, noise_dropout, temperature, log_every_t):
        model = self.model
        device = torch.device(model.device)
        # window fusion (lib/model_zoo/panorama.py): refuse unsupported inputs before any device work
        win = None
        if x_info.get('windows', None) is not None:
            from .panorama import check_sample_inputs
            win = check_sample_inputs(x_info, shape, c_infos)
        # Prompt-to-Prompt (lib/model_zoo/prompt_edit.py): refuse unsupported inputs before any device work
        pe_ctx = pe = None
        if any(ci.get('prompt_edit', None) is not None for ci in c_infos):
            from .prompt_edit import check_sample_inputs
            pe_ctx, pe = check_sample_inputs(x_info, shape, c_infos)
        # a walk from an inversion (lib/model_zoo/edit.py): its mask blends against the trajectory, with no draws
        from_inv = x_info.get('inversion', None) is not None
        if from_inv:
            from .edit import check_sample_inputs
            inv, inv_mask = check_sample_inputs(x_info, shape, self.ddim_timesteps)
        inv_blend = from_inv and inv_mask is not None
        # inpainting (lib/model_zoo/inpaint.py): refuse bad inputs before any device work; the Philox key comes from torch's CPU
        # generator, drawn only when a mask is given
        inpaint = x_info.get('inpaint_mask', None) is not None and not from_inv
        if inpaint:
            from .inpaint import check_inputs
            x0_in, mask_in = check_inputs(x_info, shape)
            seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)
        if device.type != 'cuda':
            raise RuntimeError("DDIMSampler: the H100 build has no CPU path (model.to('cuda') first)")
        ops = _ops()
        dtype = c_infos[0]['conditioning'].dtype
        bs = shape[0]
        full_walk = inpaint and x_info.get('x0_forward_timesteps', None) is None
        start_info = x_info
        if full_walk:       # a masked full walk starts from x_T as an unmasked one does, never from the img2img start
            start_info = {k: v for k, v in x_info.items() if k != 'x0'}
        elif inpaint:       # the img2img start noises x0 row by row: a batch-1 x0 is noised once per item
            start_info = dict(x_info, x0=x0_in.expand(bs, *x0_in.shape[1:]))
        elif pe is not None:    # every prompt starts from the same noise: one draw, or the given x_T, expanded to the n rows
            xt = x_info.get('xt', None)
            if xt is None:
                xt = torch.randn([1] + list(shape[1:]), device=device, dtype=dtype)
            start_info = dict(x_info, xt=xt.expand(list(shape)))
        x, timesteps = self._initial_latent(shape, start_info, dtype, device)
        x_info['x'] = x
        scale = float(c_infos[0]['unconditional_guidance_scale'])
        cfg = scale != 1.
        total_steps = timesteps.shape[0]
        if total_steps <= 0 or total_steps > 1000:
            # x0_forward_timesteps == 0 leaves no step to run: the reference's loop never executes and it raises on the unbound
            # result (ddim.py:105-127); here the device tables would be indexed at -1
            raise ValueError(f"DDIM walk of {total_steps} steps: need 1..1000 (x0_forward_timesteps must be >= 1)")
        sigmas = np.asarray(self.ddim_sigmas.cpu() if isinstance(self.ddim_sigmas, torch.Tensor) else self.ddim_sigmas)
        fast = self.use_cuda_graph and noise_dropout == 0. and not np.any(sigmas[:total_steps] != 0)

        x_type = x_info['type']
        ctxs, c_types, ratios, time_from, mch = self._contexts(c_infos, cfg, x_type, multi)
        B = 2 * bs if cfg else bs
        # text latents ([n, 768], the i2t / t2t flows: app.py:384-434) walk the same loop as a 1x1 "image" of 768 channels: the
        # NCHW <-> NHWC conversions are identities and the 0-D diffuser takes the flat view
        flat = len(shape) == 2
        H, W = (1, 1) if flat else (shape[2], shape[3])
        if flat:
            x = x.reshape(bs, shape[1], 1, 1)

        # device-side per-step tables, indexed by the DDIM index (total_steps-1 ... 0)
        coef = torch.tensor(self._coef_table(timesteps, sigmas), dtype=torch.float32, device=device).contiguous()
        ts_table = torch.tensor(np.asarray(timesteps, dtype=np.int64), device=device)

        st = self._state(bs, B, H, W, shape[1], device)
        ops.nchw_to_nhwc(x.float().contiguous(), out=st['x_in'][:bs])
        if inpaint:
            mask_per_item = self._inpaint_state(st, x0_in, mask_in, seed, total_steps, x if full_walk else None, bs, device)
        if inv_blend:
            mask_per_item = self._inversion_blend_state(st, inv, inv_mask, device)
        if pe is not None:
            pe_state = self._prompt_edit_state(st, pe, c_infos[pe_ctx], ctxs, pe_ctx, cfg, H, W, total_steps, device)
        sig_types, sig_ctxs = c_types, ctxs
        if win is not None:
            from . import panorama
            per = panorama.WINDOWS_PER_CHUNK
            chunks = win.chunks(per)
            ws = self._window_state(st, win, per, bs, cfg, shape[1], device)
            wctxs = {k: self._contexts(c_infos, cfg, x_type, multi, buffer_tag=('windows', k), repeat=k)[0]
                     for k in sorted({k for _, k in chunks})}
            sig_types = [ct for _ in wctxs for ct in c_types]
            sig_ctxs = [c for k in wctxs for c in wctxs[k]]
        if cfg:
            st['x_in'][bs:].copy_(st['x_in'][:bs])
        st['coef'][:total_steps].copy_(coef)
        st['ts'][:total_steps].copy_(ts_table)
        st['idx'].fill_(total_steps - 1)

        def windowed_eps():
            """gather -> UNet -> merge per chunk of windows, into the canvas eps [e_u; e_c]"""
            t_emb = ops.timestep_embedding(st['ts'], mch, step_idx=st['idx'], batch=ws.xw.shape[0])
            for first, k in chunks:
                rows = k * bs
                xw = ws.xw[:B // bs * rows]
                ops.window_gather(st['x_in'][:bs], ws.oy, ws.ox, win.h, win.w, first, k, out=xw[:rows],
                                  out_dup=xw[rows:] if cfg else None)
                e = model.eps_nhwc(xw, x_type, t_emb[:xw.shape[0]], c_types, wctxs[k], ratios, time_from)
                ops.window_merge(e, ws.oy, ws.ox, ws.cover_y, ws.cover_x, first, k, ws.eps, halves=B // bs)
            return ws.eps

        def step(noise=None):
            if win is not None:
                eps = windowed_eps()
            else:
                t_emb = ops.timestep_embedding(st['ts'], mch, step_idx=st['idx'], batch=B)
                eps = model.eps_nhwc(st['x_in'].view(B, -1) if flat else st['x_in'], x_type, t_emb, c_types, ctxs, ratios,
                                     time_from)
            if flat:
                eps = eps.view(B, 1, 1, -1)
            e_u, e_c = (eps[:bs], eps[bs:]) if cfg else (None, eps)
            self._update(st, e_u, e_c, scale, bs, cfg, noise, temperature)
            if inpaint:
                ops.inpaint_blend(st['x_in'][:bs], st['x0'], st['mask'] if mask_per_item else st['mask'][:1], st['blend'],
                                  st['idx'], seed=st['seed'], x_dup=st['x_in'][bs:] if cfg else None)
            if inv_blend:
                ops.inversion_blend(st['x_in'][:bs], st['traj'], st['mask'] if mask_per_item else st['mask'][:1], st['idx'],
                                    x_dup=st['x_in'][bs:] if cfg else None)
            if pe is not None and pe_state.blend:
                ops.local_blend(st['x_in'][:bs], pe_state.map, pe_state.flags, st['idx'], pe_state.h4, pe_state.w4,
                                pe_state.threshold, x_dup=st['x_in'][bs:] if cfg else None)
            ops.add_int(st['idx'], -1)

        intermediates = {'pred_xt': [], 'pred_x0': []}

        def log(index):
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates['pred_xt'].append(ops.nhwc_to_nchw(st['x_in'][:bs].contiguous()).to(dtype))
                intermediates['pred_x0'].append(ops.nhwc_to_nchw(st['pred_x0']).to(dtype))

        if not fast:
            for i in range(total_steps):
                index = total_steps - i - 1
                noise = None
                if sigmas[index] != 0:
                    noise = noise_like(st['x_in'][:bs], False)
                    if noise_dropout > 0.:
                        noise = torch.nn.functional.dropout(noise, p=noise_dropout)
                step(noise)
                log(index)
        else:
            from .diffusion_utils import pack_epoch
            key = (pack_epoch(), bs, B, H, W, x_type, tuple(c_types), tuple(ratios), scale, float(temperature), time_from,
                   tuple((c.data.data_ptr(), tuple(c.data.shape), c.length) for c in ctxs)) + self._graph_tag()
            if inpaint:
                key += (('inpaint', mask_per_item),)
            if inv_blend:
                key += (('inversion', mask_per_item),)
            if pe is not None:
                key += (('prompt_edit', pe.n, pe.has_beta, pe.blend is not None, pe_state.threshold),)
            if win is not None:
                key += (('windows', win.key(), per, tuple((c.data.data_ptr(), tuple(c.data.shape)) for c in sig_ctxs)),)
            n = self._walk(key, '_graphs', step, total_steps, st, sig_types, sig_ctxs, lambda i: log(total_steps - i - 1))
            if n is not None:
                self.last_step_launches = n

        pred_xt = ops.nhwc_to_nchw(st['x_in'][:bs].contiguous()).to(dtype)
        if flat:
            pred_xt = pred_xt.reshape(bs, -1)
            intermediates = {k: [v.reshape(bs, -1) for v in vs] for k, vs in intermediates.items()}
        x_info['x'] = pred_xt
        return pred_xt, intermediates

    def _contexts(self, c_infos, cfg, x_type, multi, buffer_tag=None, repeat=1):
        """[uncond ; cond] of every context, built once (the reference re-concatenates every step, ddim.py:146), in persistent
        padded buffers (per buffer_tag, so the inversion and the window chunks keep their own) -> (contexts, c_types, ratios,
        time_from, model_channels).  repeat = k: each half's rows repeated k times, [u; u; ...; c; c; ...], the contexts of a
        chunk of k windows (lib/model_zoo/panorama.py)."""
        from .attention import PaddedContext
        ctxs = []
        for i, ci in enumerate(c_infos):
            c = torch.cat([ci['unconditional_conditioning'], ci['conditioning']]) if cfg else ci['conditioning']
            ci['c'] = c
            if repeat != 1:
                c = torch.cat([h.repeat(repeat, 1, 1) for h in c.chunk(2 if cfg else 1)])
            ctxs.append(PaddedContext(self._ctx_buffer(i if buffer_tag is None else (buffer_tag, i), c), c.shape[1]))
        c_types = [ci['type'] for ci in c_infos]
        ratios = [float(ci.get('ratio', 1.0)) for ci in c_infos]
        time_from = self.model.time_source(x_type, multi)
        return ctxs, c_types, ratios, time_from, self.model.diffuser[time_from].model_channels

    def _walk(self, key, graphs_attr, step, total_steps, st, c_types, ctxs, log):
        """Run total_steps steps of `step` on a captured step graph kept in self.<graphs_attr>; log(i) after walk position i.
        -> the launches of one step, or None when a cached graph replayed every step."""
        model, ops = self.model, _ops()
        ent = getattr(self, graphs_attr).get(key)
        if ent is not None and ent[1] == model.context_kv_signature(c_types, ctxs):
            # steady state: the context projections were just refreshed in place; every step is a graph replay
            for i in range(total_steps):
                ent[0].replay()
                log(i)
            return None
        n0 = ops.launch_count()
        step()                      # first step eager: packs weights, sizes workspaces, warms caches
        launches = ops.launch_count() - n0
        log(0)
        g = None
        if total_steps > 1:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            idx_before = st['idx'].clone()
            x_before = st['x_in'].clone()
            with torch.cuda.graph(g):
                step()
            # capture does not execute; make sure state is exactly what the eager step left
            st['idx'].copy_(idx_before)
            st['x_in'].copy_(x_before)
            # keep one live graph (its private pool holds the activations) + the K / V^T buffers it reads
            setattr(self, graphs_attr, {key: (g, model.context_kv_signature(c_types, ctxs))})
        for i in range(1, total_steps):
            g.replay()
            log(i)
        return launches

    # ------------------------------------------------------------------ DDIM inversion (lib/model_zoo/edit.py)
    @torch.no_grad()
    def invert(self, steps, x0, c_info, k=None, verbose=False):
        """Run the DDIM ODE backwards from the image latent x0 over the first k grid points (all by default) -> Inversion."""
        return self._invert(steps, x0, [c_info], False, k, verbose)

    @torch.no_grad()
    def invert_multicontext(self, steps, x0, c_info_list, k=None, verbose=False):
        scale = c_info_list[0]['unconditional_guidance_scale']
        for ci in c_info_list:
            assert scale == ci['unconditional_guidance_scale'], \
                "A different unconditional guidance scale between different context is not allowed!"
        return self._invert(steps, x0, c_info_list, True, k, verbose)

    def _invert(self, steps, x0, c_infos, multi, k, verbose):
        from .edit import Inversion, check_invert_inputs, context_batch, inversion_rows
        model = self.model
        device = torch.device(model.device)
        self.make_schedule(ddim_num_steps=steps, ddim_eta=0., verbose=verbose)
        timesteps = self.ddim_timesteps
        bs = context_batch(c_infos, float(c_infos[0]['unconditional_guidance_scale']))
        k = check_invert_inputs(x0, bs, k, len(timesteps))
        if device.type != 'cuda':
            raise RuntimeError("DDIMSampler: the H100 build has no CPU path (model.to('cuda') first)")
        ops = _ops()
        _, C, H, W = x0.shape
        scale = float(c_infos[0]['unconditional_guidance_scale'])
        cfg = scale != 1.
        B = 2 * bs if cfg else bs
        ctxs, c_types, ratios, time_from, mch = self._contexts(c_infos, cfg, 'image', multi, buffer_tag='invert')
        st = self._inv_state(bs, B, H, W, C, len(timesteps) + 1, device)
        ring = st['ring']
        ring[0].copy_(ops.nchw_to_nhwc(x0.to(device=device, dtype=torch.float32).expand(bs, C, H, W).contiguous()))
        st['x_in'][:bs].copy_(ring[0])
        if cfg:
            st['x_in'][bs:].copy_(ring[0])
        st['coef'][:k].copy_(torch.from_numpy(inversion_rows(self.ddim_alphas, self.ddim_alphas_prev, k)))
        st['ts'][:len(timesteps)].copy_(torch.tensor(np.asarray(timesteps, dtype=np.int64)))
        st['idx'].fill_(0)

        def step():
            t_emb = ops.timestep_embedding(st['ts'], mch, step_idx=st['idx'], batch=B)
            eps = model.eps_nhwc(st['x_in'], 'image', t_emb, c_types, ctxs, ratios, time_from)
            e_u, e_c = (eps[:bs], eps[bs:]) if cfg else (None, eps)
            DDIMSampler._update(self, st, e_u, e_c, scale, bs, cfg, None, 1.0)
            ops.latent_store_slot(st['x_in'][:bs], ring, st['idx'], 1)
            ops.add_int(st['idx'], 1)

        if not self.use_cuda_graph:
            for _ in range(k):
                step()
        else:
            from .diffusion_utils import pack_epoch
            key = (pack_epoch(), bs, B, H, W, tuple(c_types), tuple(ratios), scale, time_from,
                   tuple((c.data.data_ptr(), tuple(c.data.shape), c.length) for c in ctxs), 'invert')
            n = self._walk(key, '_inv_graphs', step, k, st, c_types, ctxs, lambda i: None)
            if n is not None:
                self.last_invert_step_launches = n
        return Inversion(ring[:k + 1].clone(), steps, k, timesteps, (bs, C, H, W))

    # ------------------------------------------------------------------ per-step update (overridden by DPMSolverSampler)
    _coef_cols = 4      # width of a row of the device coefficient table

    def _coef_table(self, timesteps, sigmas):
        """fp32 [len(timesteps), 4] rows {a_t, a_prev, sigma_t, sqrt(1 - a_t)} of the walk, indexed by the DDIM index."""
        total_steps = timesteps.shape[0]
        return np.stack([np.asarray(self.ddim_alphas.cpu() if isinstance(self.ddim_alphas, torch.Tensor) else self.ddim_alphas, dtype=np.float32)[:total_steps],
                         np.asarray(self.ddim_alphas_prev, dtype=np.float32)[:total_steps],
                         sigmas.astype(np.float32)[:total_steps],
                         np.asarray(self.ddim_sqrt_one_minus_alphas.cpu() if isinstance(self.ddim_sqrt_one_minus_alphas, torch.Tensor) else self.ddim_sqrt_one_minus_alphas, dtype=np.float32)[:total_steps]], axis=1)

    def _update(self, st, e_u, e_c, scale, bs, cfg, noise, temperature):
        """CFG mix + x_{t-1} from row st['idx'] of st['coef']: x_in[:bs] in place, its copy into x_in[bs:], pred_x0."""
        _ops().ddim_cfg_step(e_u, e_c, st['x_in'][:bs], st['coef'], scale, x_prev=st['x_in'][:bs],
                             x_prev_dup=st['x_in'][bs:] if cfg else None, pred_x0=st['pred_x0'], noise=noise,
                             temperature=temperature, step_idx=st['idx'])

    def _graph_tag(self):
        """What else, besides the shapes and contexts, the captured step graph depends on."""
        return ()

    def _ctx_buffer(self, i, c):
        """Persistent zero-padded bf16 copy of context i ([B, L, C] -> [B, ceil8(L), C]); refilled in place."""
        bufs = self.__dict__.setdefault('_ctx_bufs', {})
        B, L, Cc = c.shape
        Lp = (L + 7) // 8 * 8
        buf = bufs.get(i)
        if buf is None or tuple(buf.shape) != (B, Lp, Cc) or buf.device != c.device:
            buf = torch.zeros(B, Lp, Cc, dtype=torch.bfloat16, device=c.device)
            bufs[i] = buf
        buf[:, :L].copy_(c)
        return buf

    def _state(self, bs, B, H, W, C, device):
        key = (bs, B, H, W, C, str(device))
        st = getattr(self, '_st', None)
        if st is None or st['key'] != key:
            st = {'key': key,
                  'x_in': torch.zeros(B, H, W, C, dtype=torch.float32, device=device),
                  'pred_x0': torch.zeros(bs, H, W, C, dtype=torch.float32, device=device),
                  'coef': torch.zeros(1000, self._coef_cols, dtype=torch.float32, device=device),
                  'ts': torch.zeros(1000, dtype=torch.int64, device=device),
                  'idx': torch.zeros(1, dtype=torch.int32, device=device)}
            self._st = st
            self._graphs = {}
        return st

    def _inv_state(self, bs, B, H, W, C, slots, device):
        """The inversion walk's own persistent buffers (so it never evicts the sampling graph) and its trajectory ring."""
        key = (bs, B, H, W, C, slots, str(device))
        st = getattr(self, '_inv_st', None)
        if st is None or st['key'] != key:
            st = {'key': key,
                  'x_in': torch.zeros(B, H, W, C, dtype=torch.float32, device=device),
                  'pred_x0': torch.zeros(bs, H, W, C, dtype=torch.float32, device=device),
                  'coef': torch.zeros(1000, 4, dtype=torch.float32, device=device),
                  'ts': torch.zeros(1000, dtype=torch.int64, device=device),
                  'idx': torch.zeros(1, dtype=torch.int32, device=device),
                  'ring': torch.zeros(slots, bs, H, W, C, dtype=torch.float32, device=device)}
            self._inv_st = st
            self._inv_graphs = {}
        return st

    def _inversion_blend_state(self, st, inv, mask, device):
        """Refill the trajectory and mask buffers of st in place, so a cached step graph replays on a new inversion and mask ->
        whether the mask is per item.  lib/model_zoo/edit.py specifies the semantics."""
        ops = _ops()
        bs, H, W = inv.bs, inv.shape[2], inv.shape[3]
        traj = st.get('traj')
        if traj is None or traj.shape[0] < inv.k or tuple(traj.shape[1:]) != tuple(inv.trajectory.shape[1:]):
            st['traj'] = torch.zeros((max(inv.k, len(self.ddim_timesteps)),) + tuple(inv.trajectory.shape[1:]),
                                     dtype=torch.float32, device=device)
            self._graphs = {}           # a cached graph reads the old buffer
        st['traj'][:inv.k].copy_(inv.trajectory[:inv.k])
        if 'mask' not in st:
            st['mask'] = torch.zeros(bs, H * W, dtype=torch.float32, device=device)
        mask = mask.to(device=device, dtype=torch.float32).contiguous()
        if mask.shape[-1] != W:
            mask = ops.mask_to_latent(mask)
        st['mask'][:mask.shape[0]].copy_(mask.view(mask.shape[0], H * W))
        return int(mask.shape[0] != 1)

    def _prompt_edit_state(self, st, ed, ci, ctxs, i, cfg, H, W, total_steps, device):
        """Swap context i for its persistent extended buffer [context rows; edited contexts] and refill the edit's device state
        in st in place, so a cached step graph replays on new prompts and tables -> the prompt_edit.EditState (also carried
        by the context).  lib/model_zoo/prompt_edit.py specifies the semantics."""
        from .attention import PaddedContext
        from .prompt_edit import EditState, quarter
        c = ci['c']
        ext = torch.cat([c.float(), ed.edited_contexts(ci['conditioning']).to(c.device)])
        buf = self._ctx_buffer(('prompt_edit', i), ext)
        es = st.get('prompt_edit')
        want = (ed.n, 2 * ed.n if cfg else ed.n, ext.shape[0], ed.has_beta, ed.blend is not None, quarter(H), quarter(W))
        if es is None or es.key() != want:
            es = EditState(ed.n, cfg, ext.shape[0], ed.has_beta, ed.blend is not None, quarter(H), quarter(W), device)
            st['prompt_edit'] = es
            self._graphs = {}           # a cached graph reads the old buffers
        es.fill(ed, total_steps, cfg, st['idx'])
        ctxs[i] = PaddedContext(buf, c.shape[1], edit=es)
        return es

    def _window_state(self, st, lay, per, bs, cfg, C, device):
        """The persistent device state of a windowed walk in st (panorama.WindowState), its layout tables refilled in place, so a
        cached step graph replays on new prompts or a new x_T.  lib/model_zoo/panorama.py specifies the semantics."""
        from .panorama import WindowState
        ws = st.get('windows')
        if ws is None or ws.key != WindowState.key_for(lay, per, bs, cfg, C):
            ws = WindowState(lay, per, bs, cfg, C, device)
            st['windows'] = ws
            self._graphs = {}           # a cached graph reads the old buffers
        ws.fill(lay)
        return ws

    def _inpaint_state(self, st, x0, mask, seed, total_steps, x_T, bs, device):
        """Refill the inpainting buffers of st in place, so a cached step graph replays on a new image, mask and seed ->
        whether the mask is per item.  With x_T (the full walk) the kept region of x_in[:bs] becomes x0 noised to t_top with
        x_T's own draw.  lib/model_zoo/inpaint.py specifies the semantics."""
        from .inpaint import blend_table
        ops = _ops()
        _, H, W, C = st['x_in'].shape
        if 'x0' not in st:
            st.update(x0=torch.zeros(bs, H, W, C, dtype=torch.float32, device=device),
                      mask=torch.zeros(bs, H * W, dtype=torch.float32, device=device),
                      blend=torch.zeros(1000, 2, dtype=torch.float32, device=device),
                      seed=torch.zeros(1, dtype=torch.int64, device=device))
        st['x0'].copy_(ops.nchw_to_nhwc(x0.to(device=device, dtype=torch.float32).contiguous()))   # broadcasts a [1] batch
        mask = mask.to(device=device, dtype=torch.float32).contiguous()
        if mask.shape[-1] != W:
            mask = ops.mask_to_latent(mask)
        st['mask'][:mask.shape[0]].copy_(mask.view(mask.shape[0], H * W))
        st['blend'][:total_steps].copy_(torch.from_numpy(blend_table(self.ddim_alphas_prev[:total_steps])))
        st['seed'].copy_(seed)
        mask_per_item = int(mask.shape[0] != 1)
        if x_T is not None:
            a_top = float(self.ddim_alphas[total_steps - 1])
            row = torch.tensor([[np.sqrt(a_top), np.sqrt(1.0 - a_top)]], dtype=torch.float32, device=device)
            ops.inpaint_blend(st['x_in'][:bs], st['x0'], st['mask'] if mask_per_item else st['mask'][:1], row,
                              torch.zeros(1, dtype=torch.int32, device=device),
                              noise=ops.nchw_to_nhwc(x_T.float().contiguous()))
        return mask_per_item

    # ------------------------------------------------------------------ single-step API (reference parity)
    @torch.no_grad()
    def p_sample_ddim(self, x_info, c_info, t, index, repeat_noise=False, use_original_steps=False,
                      noise_dropout=0., temperature=1.):
        return self._p_sample(x_info, [c_info], False, t, index, repeat_noise, use_original_steps, noise_dropout,
                              temperature)

    @torch.no_grad()
    def p_sample_ddim_multicontext(self, x_info, c_info_list, t, index, repeat_noise=False,
                                   use_original_steps=False, noise_dropout=0., temperature=1.):
        return self._p_sample(x_info, c_info_list, True, t, index, repeat_noise, use_original_steps, noise_dropout,
                              temperature)

    def _p_sample(self, x_info, c_infos, multi, t, index, repeat_noise, use_original_steps, noise_dropout, temperature):
        """One eager DDIM step with the reference's argument conventions (ddim.py:129-171, 244-298)."""
        if any(ci.get('prompt_edit', None) is not None for ci in c_infos):
            raise NotImplementedError("a prompt edit spans the walk (its windows and word maps): use sample / "
                                      "sample_multicontext (lib/model_zoo/prompt_edit.py)")
        if x_info.get('windows', None) is not None:
            raise NotImplementedError("window fusion runs inside the sampler's walk: use sample / sample_multicontext "
                                      "(lib/model_zoo/panorama.py)")
        ops = _ops()
        model = self.model
        x = x_info['x']
        require_cuda(x, "DDIMSampler.p_sample_ddim")
        scale = c_infos[0]['unconditional_guidance_scale']
        for ci in c_infos:
            assert scale == ci['unconditional_guidance_scale'], \
                "A different unconditional guidance scale between different context is not allowed!"
        cfg = scale != 1.
        for ci in c_infos:
            ci['c'] = torch.cat([ci['unconditional_conditioning'], ci['conditioning']]) if cfg else ci['conditioning']
        x_in, t_in = (torch.cat([x] * 2), torch.cat([t] * 2)) if cfg else (x, t)
        x_info['x'] = x_in
        e = model.apply_model_multicontext(x_info, t_in, c_infos) if multi else model.apply_model(x_info, t_in, c_infos[0])
        e_u, e_c = e.float().chunk(2) if cfg else (None, e.float())
        alphas = model.alphas_cumprod if use_original_steps else self.ddim_alphas
        alphas_prev = model.alphas_cumprod_prev if use_original_steps else self.ddim_alphas_prev
        s1m = model.sqrt_one_minus_alphas_cumprod if use_original_steps else self.ddim_sqrt_one_minus_alphas
        sigmas = self.ddim_sigmas_for_original_num_steps if use_original_steps else self.ddim_sigmas
        coef = torch.tensor([[float(alphas[index]), float(alphas_prev[index]), float(sigmas[index]), float(s1m[index])]],
                            dtype=torch.float32, device=x.device)
        noise = None
        if float(sigmas[index]) != 0:
            noise = noise_like(x, repeat_noise).float()
            if noise_dropout > 0.:
                noise = torch.nn.functional.dropout(noise, p=noise_dropout)
        pred_x0 = torch.empty_like(x, dtype=torch.float32)
        x_prev, _ = ops.ddim_cfg_step(None if e_u is None else e_u.contiguous(), e_c.contiguous(), x.float().contiguous(),
                                      coef, scale, pred_x0=pred_x0, noise=None if noise is None else noise.contiguous(),
                                      temperature=temperature)
        return x_prev.to(x.dtype), pred_x0.to(x.dtype)
