"""DDIMSampler on vdb200 kernels — same public surface as the reference (lib/model_zoo/ddim.py:10-298):
make_schedule, sample, ddim_sampling, p_sample_ddim and the *_multicontext twins.

Fast path (eta == 0, no noise dropout): the whole DDIM step — sinusoid, time MLP, all ResBlock emb
projections, the 46-block UNet walk over the CFG-doubled batch, and the fused CFG + x_{t-1} update —
is captured ONCE as a CUDA graph whose per-step scalars (timestep, a_t, a_prev, sigma, sqrt(1-a_t))
live in device tables indexed by a device-side step counter; the 50-step loop is 50 graph replays with
no host<->device traffic (the reference does ~15 tiny kernels + 4 H2D fills per step, ddim.py:159-171).
The latent stays fp32 NHWC between steps; NCHW conversion happens only at the API boundary.
"""
from types import SimpleNamespace

import numpy as np
import torch

from .diffusion_utils import (GRIDS, make_ddim_sampling_parameters, make_ddim_timesteps, noise_like, pack_epoch,
                              require_cuda, to_numpy)


def _ops():
    from vdb200 import ops
    return ops


# ------------------------------------------------------------------ sampling modes and how they combine
# A mode is selected by an optional input: x_info['sag'] (lib/model_zoo/sag.py), x_info['regions'] (regions.py), x_info['windows']
# (panorama.py: the region walk with no regions), a context's 'prompt_edit' (prompt_edit.py), x_info['inversion'] (edit.py) and
# x_info['inpaint_mask'] (inpaint.py).  The start inputs x_info['x0'] (with
# 'x0_forward_timesteps') and x_info['xt'] select no mode, but some modes refuse them.
#
# REFUSES: who -> {input given: (exception type, message)}, checked in this order.
#   - Entry points, before anything else: 'sample' (DDIMSampler's and DPMSolverSampler's sample / sample_multicontext), 'plms'
#     (PLMSSampler's) and 'p_sample' (p_sample_ddim(_multicontext), which ignores the inputs it does not list).
#   - Modes, for the pairs that refuse each other: each mode checks its row after the type of its own input and before its
#     other checks, modes in the order of DDIMSampler._modes.
REFUSES = {
    'sample': {},
    'plms': {k: (NotImplementedError, msg) for k, msg in (
        ('inpaint_mask', "PLMSSampler has no inpainting: use DDIMSampler or DPMSolverSampler (lib/model_zoo/inpaint.py)"),
        ('prompt_edit', "PLMSSampler has no prompt editing: use DDIMSampler or DPMSolverSampler (lib/model_zoo/prompt_edit.py)"),
        ('windows', "PLMSSampler has no window fusion: use DDIMSampler or DPMSolverSampler (lib/model_zoo/panorama.py)"),
        ('regions', "PLMSSampler has no region prompts: use DDIMSampler or DPMSolverSampler (lib/model_zoo/regions.py)"),
        ('inversion', "PLMSSampler cannot sample from an inversion: use DDIMSampler or DPMSolverSampler "
                      "(lib/model_zoo/edit.py)"),
        ('sag', "PLMSSampler has no self-attention guidance: use DDIMSampler or DPMSolverSampler (lib/model_zoo/sag.py)"))},
    'p_sample': {
        'prompt_edit': (NotImplementedError, "a prompt edit spans the walk (its windows and word maps): use sample / "
                                             "sample_multicontext (lib/model_zoo/prompt_edit.py)"),
        'windows': (NotImplementedError, "window fusion runs inside the sampler's walk: use sample / sample_multicontext "
                                         "(lib/model_zoo/panorama.py)"),
        'regions': (NotImplementedError, "region prompts run inside the sampler's walk: use sample / sample_multicontext "
                                         "(lib/model_zoo/regions.py)"),
        'sag': (NotImplementedError, "self-attention guidance runs inside the sampler's walk: use sample / sample_multicontext "
                                     "(lib/model_zoo/sag.py)")},
    'sag': {
        'windows': (NotImplementedError, "SAG with windows: window fusion replaces the UNet call (lib/model_zoo/sag.py)"),
        'regions': (NotImplementedError, "SAG with regions: region prompts replace the UNet call (lib/model_zoo/sag.py)"),
        'prompt_edit': (NotImplementedError, "SAG with prompt_edit: the edit's item tables index the CFG batch and know nothing of "
                                             "SAG's second pass (lib/model_zoo/sag.py)")},
    'regions': {
        'prompt_edit': (NotImplementedError, "regions with prompt_edit: the edit's item tables index prompts, not regions "
                                             "(lib/model_zoo/regions.py)"),
        'inversion': (NotImplementedError, "regions cannot sample from an inversion (lib/model_zoo/regions.py)")},
    'windows': {
        'prompt_edit': (NotImplementedError, "windows with prompt_edit: the edit's item tables index prompts, not windows "
                                             "(lib/model_zoo/panorama.py)"),
        'inversion': (NotImplementedError, "windows cannot sample from an inversion (lib/model_zoo/panorama.py)")},
    'prompt_edit': {k: (ValueError, f"'prompt_edit' does not combine with {k!r}") for k in ('x0', 'inpaint_mask', 'inversion')},
    'inversion': {k: (ValueError, f"x_info['{k}'] cannot be given with 'inversion': the walk starts from the inversion")
                  for k in ('xt', 'x0', 'x0_forward_timesteps')},
}

# Pairs that change meaning: mode -> inputs it takes over, which then select no mode of their own.  An inpaint_mask given with an
# inversion is the mask of the inversion's trajectory blend, not inpainting.  Windows given with regions are the region walk's
# window layout, not a walk of their own.
TAKES = {'inversion': ('inpaint_mask',), 'regions': ('windows',)}


def given_inputs(x_info, c_infos):
    """The optional inputs given (not None) to a call."""
    given = {k for k in ('x0', 'xt', 'x0_forward_timesteps', 'inpaint_mask', 'inversion', 'windows', 'regions', 'sag')
             if x_info.get(k, None) is not None}
    if any(ci.get('prompt_edit', None) is not None for ci in c_infos):
        given.add('prompt_edit')
    return given


def refuse(who, x_info, c_infos):
    """Raise what REFUSES says `who` (an entry point or a mode) raises for the inputs given."""
    given = given_inputs(x_info, c_infos)
    for k, (exc, msg) in REFUSES[who].items():
        if k in given:
            raise exc(msg)


def buffers_key(*bufs):
    """The identity (address and shape) of the device buffers a captured step graph reads, for its key."""
    return tuple((b.data_ptr(), tuple(b.shape)) for b in bufs if b is not None)


class SamplerMode(object):
    """A mode's part in DDIMSampler's walk.  The constructor checks the mode's inputs on the host, before any device work; the
    mode keeps its persistent device state in the walk record (run.walk, under the mode's own names), refilled in place so a
    cached step graph replays.  `run` is the call's record (DDIMSampler._run): the walk record, the batch and latent shape, the contexts, and
    run.x / run.x_dup, the latent [bs, H, W, C] and its CFG duplicate (or None)."""

    def start(self, sampler, x_info, shape, dtype, device):
        """-> (x_T NCHW, the grid points to walk) when the mode changes the start latent, else None."""
        return None

    def prepare(self, sampler, run):
        """Refill the device state for this call (a mode may also swap the contexts the step reads) -> its part of the graph
        key, which covers every buffer the mode's launches read."""
        raise NotImplementedError

    def eps(self, sampler, run):
        """-> the step's eps [run.B, H, W, C] when the mode replaces the UNet call on the latent, else None."""
        return None

    def after_update(self, run):
        """The mode's launches after the step's update, before the step counter moves."""


class _Walk(dict):
    """The persistent device buffers of one kind of walk by name (sampling or inversion, so neither evicts the other's graph),
    with the device state its modes add, and `graphs`, its one captured step graph as {key: (CUDAGraph, K / V^T signature)}
    (one live graph: its private pool holds the activations).  The graph reads these buffers, so it lives and dies with the
    record."""

    def __init__(self, key, bs, B, H, W, C, cols, rings, device):
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=device)
        super().__init__(x_in=z(B, H, W, C), pred_x0=z(bs, H, W, C), coef=z(1000, cols), ts=z(1000, dtype=torch.int64),
                         idx=z(1, dtype=torch.int32), **{name: z(*s) for name, s in rings.items()})
        self.key, self.graphs = key, {}


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        super().__init__()
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.use_cuda_graph = kwargs.get("use_cuda_graph", True)
        # the time grid every walk of this sampler takes (make_ddim_timesteps): 'uniform' (DDIM's), 'trailing' or 'karras'
        self.grid = kwargs.get("grid", "uniform")
        if self.grid not in GRIDS:
            raise ValueError(f"grid must be one of {GRIDS}, got {self.grid!r}")

    def register_buffer(self, name, attr):
        # the reference forces .to('cuda') here (ddim.py:17-21); follow the model's device instead
        if isinstance(attr, torch.Tensor) and str(self.model.device) != 'cpu' and attr.device != torch.device(self.model.device):
            attr = attr.to(torch.device(self.model.device))
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize=None, ddim_eta=0., verbose=True):
        """reference ddim.py:23-56 (same fp64/fp32 dtype walk).  ddim_discretize defaults to the sampler's grid."""
        self.ddim_timesteps = make_ddim_timesteps(ddim_discr_method=ddim_discretize or self.grid,
                                                  num_ddim_timesteps=ddim_num_steps, num_ddpm_timesteps=self.ddpm_num_timesteps,
                                                  verbose=verbose, alphas_cumprod=self.model.alphas_cumprod)
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
        """ddim.py:94-105: injected x_T ('xt'), img2img start (x0 + q_sample) or fresh noise."""
        timesteps = self.ddim_timesteps
        if x_info.get('xt', None) is not None:
            x = x_info['xt'].to(dtype).to(device)       # (the reference's `.astype` here is a bug, ddim.py:95)
        elif x_info.get('x0', None) is not None:
            k = x_info['x0_forward_timesteps']
            if k >= len(timesteps):
                # x0 is noised to grid point k, so k must lie on the grid, which can be shorter than the steps asked for (a
                # Karras grid drops low sigmas that round to one timestep)
                raise ValueError(f"x0_forward_timesteps must be below the grid's {len(timesteps)} points, got {k}")
            x0 = x_info['x0'].type(dtype).to(device)
            ts = np.repeat(timesteps[k], shape[0])
            ts = torch.Tensor(ts).long().to(device)
            timesteps = timesteps[:x_info['x0_forward_timesteps']]
            x = self.model.q_sample(x0, ts)
        else:
            x = torch.randn(shape, device=device, dtype=dtype)
        return x, timesteps

    def _modes(self, entry, x_info, shape, c_infos):
        """Refuse what entry point `entry` does not take, then build the active modes in the order they check their inputs
        (the order in which refusals win) -> [SamplerMode].  Host work only: every refusal comes before any device work."""
        from .edit import FromInversion
        from .inpaint import Inpainting
        from .prompt_edit import PromptEditing
        from .regions import RegionPrompts
        from .sag import SelfAttention
        refuse(entry, x_info, c_infos)
        given = given_inputs(x_info, c_infos)
        taken = {k for m in given for k in TAKES.get(m, ())}
        return [cls(self, x_info, shape, c_infos) for name, cls in (('sag', SelfAttention), ('regions', RegionPrompts),
                                                                      ('windows', RegionPrompts),
                                                                      ('prompt_edit', PromptEditing), ('inversion', FromInversion),
                                                                      ('inpaint_mask', Inpainting))
                if name in given and name not in taken]

    def _run(self, shape, x_info, c_infos, multi, noise_dropout, temperature, log_every_t):
        model = self.model
        device = torch.device(model.device)
        modes = self._modes('sample', x_info, shape, c_infos)
        if device.type != 'cuda':
            raise RuntimeError("DDIMSampler: the H100 build has no CPU path (model.to('cuda') first)")
        ops = _ops()
        dtype = c_infos[0]['conditioning'].dtype
        bs = shape[0]
        starts = [s for s in (m.start(self, x_info, shape, dtype, device) for m in modes) if s is not None]
        # REFUSES and TAKES leave at most one mode that changes the start
        x, timesteps = starts[0] if starts else self._initial_latent(shape, x_info, dtype, device)
        x_info['x'] = x
        scale = float(c_infos[0]['unconditional_guidance_scale'])
        cfg = scale != 1.
        total_steps = timesteps.shape[0]
        if total_steps <= 0 or total_steps > 1000:
            # x0_forward_timesteps == 0 leaves no step to run: the reference's loop never executes and it raises on the unbound
            # result (ddim.py:105-127); here the device tables would be indexed at -1
            raise ValueError(f"DDIM walk of {total_steps} steps: need 1..1000 (x0_forward_timesteps must be >= 1)")
        sigmas = to_numpy(self.ddim_sigmas)
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

        w = self._walk_record('_st', bs, B, H, W, shape[1], self._coef_cols, device, self._rings(bs, H, W, shape[1]))
        ops.nchw_to_nhwc(x.float().contiguous(), out=w['x_in'][:bs])
        run = SimpleNamespace(walk=w, modes=modes, bs=bs, B=B, H=H, W=W, C=shape[1], cfg=cfg, scale=scale, flat=flat,
                              total=total_steps, device=device, x_type=x_type, multi=multi, c_infos=c_infos, c_types=c_types,
                              ctxs=ctxs, ratios=ratios, time_from=time_from, mch=mch, kv_types=c_types, kv_ctxs=ctxs,
                              x=w['x_in'][:bs], x_dup=w['x_in'][bs:] if cfg else None)
        mode_keys = tuple(m.prepare(self, run) for m in modes)
        if cfg:
            w['x_in'][bs:].copy_(w['x_in'][:bs])
        w['coef'][:total_steps].copy_(coef)
        w['ts'][:total_steps].copy_(ts_table)
        w['idx'].fill_(total_steps - 1)

        def step(noise=None):
            e_u, e_c = self._eps(run)
            self._update(w, e_u, e_c, scale, bs, cfg, noise, temperature)
            for m in modes:
                m.after_update(run)
            ops.add_int(w['idx'], -1)

        intermediates = {'pred_xt': [], 'pred_x0': []}

        def log(index):
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates['pred_xt'].append(ops.nhwc_to_nchw(w['x_in'][:bs].contiguous()).to(dtype))
                intermediates['pred_x0'].append(ops.nhwc_to_nchw(w['pred_x0']).to(dtype))

        if not fast:
            for i in range(total_steps):
                index = total_steps - i - 1
                noise = None
                if sigmas[index] != 0:
                    noise = noise_like(w['x_in'][:bs], False)
                    if noise_dropout > 0.:
                        noise = torch.nn.functional.dropout(noise, p=noise_dropout)
                step(noise)
                log(index)
        else:
            n = self._walk(run, (float(temperature),) + self._graph_tag() + mode_keys, step, total_steps,
                           lambda i: log(total_steps - i - 1))
            if n is not None:
                self.last_step_launches = n

        pred_xt = ops.nhwc_to_nchw(w['x_in'][:bs].contiguous()).to(dtype)
        if flat:
            pred_xt = pred_xt.reshape(bs, -1)
            intermediates = {k: [v.reshape(bs, -1) for v in vs] for k, vs in intermediates.items()}
        x_info['x'] = pred_xt
        return pred_xt, intermediates

    def _contexts(self, c_infos, cfg, x_type, multi, buffer_tag=None):
        """[uncond ; cond] of every context, built once (the reference re-concatenates every step, ddim.py:146), in persistent
        padded buffers (per buffer_tag, so the inversion keeps its own) -> (contexts, c_types, ratios, time_from,
        model_channels)."""
        from .attention import PaddedContext
        ctxs = []
        for i, ci in enumerate(c_infos):
            c = torch.cat([ci['unconditional_conditioning'], ci['conditioning']]) if cfg else ci['conditioning']
            ci['c'] = c
            ctxs.append(PaddedContext(self._ctx_buffer(i if buffer_tag is None else (buffer_tag, i), c), c.shape[1]))
        c_types = [ci['type'] for ci in c_infos]
        ratios = [float(ci.get('ratio', 1.0)) for ci in c_infos]
        time_from = self.model.time_source(x_type, multi)
        return ctxs, c_types, ratios, time_from, self.model.diffuser[time_from].model_channels

    def _eps(self, run):
        """The step's eps at the walk's timestep, as its CFG halves (e_u or None, e_c): the UNet on the latent, or the eps of a
        mode that replaces that call."""
        w = run.walk
        for m in run.modes:
            eps = m.eps(self, run)
            if eps is not None:
                break
        else:
            t_emb = _ops().timestep_embedding(w['ts'], run.mch, step_idx=w['idx'], batch=run.B)
            eps = self.model.eps_nhwc(w['x_in'].view(run.B, -1) if run.flat else w['x_in'], run.x_type, t_emb, run.c_types,
                                      run.ctxs, run.ratios, run.time_from)
        if run.flat:
            eps = eps.view(run.B, 1, 1, -1)
        return (eps[:run.bs], eps[run.bs:]) if run.cfg else (None, eps)

    def _walk(self, run, tag, step, total_steps, log):
        """Run total_steps steps of `step` on the captured step graph kept in run.walk; log(i) after walk position i.  The key
        covers the shapes, the contexts the step reads and `tag`.  -> the launches of one step, or None when a cached graph
        replayed every step."""
        model, ops, w = self.model, _ops(), run.walk
        key = (pack_epoch(), run.bs, run.B, run.H, run.W, run.x_type, tuple(run.kv_types), tuple(run.ratios), run.scale,
               run.time_from, tuple((c.data.data_ptr(), tuple(c.data.shape), c.length) for c in run.kv_ctxs)) + tag
        ent = w.graphs.get(key)
        if ent is not None and ent[1] == model.context_kv_signature(run.kv_types, run.kv_ctxs):
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
            idx_before = w['idx'].clone()
            x_before = w['x_in'].clone()
            with torch.cuda.graph(g):
                step()
            # capture does not execute; make sure state is exactly what the eager step left
            w['idx'].copy_(idx_before)
            w['x_in'].copy_(x_before)
            # keep one live graph (its private pool holds the activations) + the K / V^T buffers it reads
            w.graphs = {key: (g, model.context_kv_signature(run.kv_types, run.kv_ctxs))}
        for i in range(1, total_steps):
            g.replay()
            log(i)
        return launches

    def _walk_record(self, attr, bs, B, H, W, C, cols, device, rings):
        """The persistent _Walk in self.<attr> ('_st' samples, '_inv_st' inverts), rebuilt (dropping its graph) when its buffers
        change shape."""
        key = (bs, B, H, W, C, cols, tuple(rings.items()), str(device))
        w = getattr(self, attr, None)
        if w is None or w.key != key:
            w = _Walk(key, bs, B, H, W, C, cols, rings, device)
            setattr(self, attr, w)
        return w

    # the cached step graph of the sampling walk and of the inversion walk, {key: (CUDAGraph, K / V^T signature)}
    _graphs = property(lambda self: self._st.graphs if hasattr(self, '_st') else {})
    _inv_graphs = property(lambda self: self._inv_st.graphs if hasattr(self, '_inv_st') else {})

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
        device = torch.device(self.model.device)
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
        w = self._walk_record('_inv_st', bs, B, H, W, C, 4, device, {'ring': (len(timesteps) + 1, bs, H, W, C)})
        ring = w['ring']
        ring[0].copy_(ops.nchw_to_nhwc(x0.to(device=device, dtype=torch.float32).expand(bs, C, H, W).contiguous()))
        w['x_in'][:bs].copy_(ring[0])
        if cfg:
            w['x_in'][bs:].copy_(ring[0])
        w['coef'][:k].copy_(torch.from_numpy(inversion_rows(self.ddim_alphas, self.ddim_alphas_prev, k)))
        w['ts'][:len(timesteps)].copy_(torch.tensor(np.asarray(timesteps, dtype=np.int64)))
        w['idx'].fill_(0)
        run = SimpleNamespace(walk=w, modes=[], bs=bs, B=B, H=H, W=W, cfg=cfg, scale=scale, flat=False, x_type='image',
                              c_types=c_types, ctxs=ctxs, ratios=ratios, time_from=time_from, mch=mch, kv_types=c_types,
                              kv_ctxs=ctxs)

        def step():
            e_u, e_c = self._eps(run)
            DDIMSampler._update(self, w, e_u, e_c, scale, bs, cfg, None, 1.0)
            ops.latent_store_slot(w['x_in'][:bs], ring, w['idx'], 1)
            ops.add_int(w['idx'], 1)

        if not self.use_cuda_graph:
            for _ in range(k):
                step()
        else:
            n = self._walk(run, (), step, k, lambda i: None)
            if n is not None:
                self.last_invert_step_launches = n
        return Inversion(ring[:k + 1].clone(), steps, k, timesteps, (bs, C, H, W))

    # ------------------------------------------------------------------ per-step update (overridden by DPMSolverSampler)
    _coef_cols = 4      # width of a row of the device coefficient table

    def _coef_table(self, timesteps, sigmas):
        """fp32 [len(timesteps), 4] rows {a_t, a_prev, sigma_t, sqrt(1 - a_t)} of the walk, indexed by the DDIM index."""
        total_steps = timesteps.shape[0]
        return np.stack([to_numpy(self.ddim_alphas, np.float32)[:total_steps],
                         np.asarray(self.ddim_alphas_prev, dtype=np.float32)[:total_steps],
                         sigmas.astype(np.float32)[:total_steps],
                         to_numpy(self.ddim_sqrt_one_minus_alphas, np.float32)[:total_steps]], axis=1)

    def _rings(self, bs, H, W, C):
        """name -> shape of the sampling walk's extra persistent buffers (DPMSolverSampler's history ring)."""
        return {}

    def _update(self, w, e_u, e_c, scale, bs, cfg, noise, temperature):
        """CFG mix + x_{t-1} from row w['idx'] of w['coef']: x_in[:bs] in place, its copy into x_in[bs:], pred_x0."""
        _ops().ddim_cfg_step(e_u, e_c, w['x_in'][:bs], w['coef'], scale, x_prev=w['x_in'][:bs],
                             x_prev_dup=w['x_in'][bs:] if cfg else None, pred_x0=w['pred_x0'], noise=noise, temperature=temperature,
                             step_idx=w['idx'])

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
        refuse('p_sample', x_info, c_infos)
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
