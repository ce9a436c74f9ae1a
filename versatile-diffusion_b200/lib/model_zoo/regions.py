"""Region prompts — MultiDiffusion region-based generation inside the captured DDIM / DPM-Solver++ step graph.

The reference has no region mode; this is an addition, and its semantics are specified here.  A region prompt says where a prompt
applies: "a red car on the left, a pine forest on the right, a snowy sky above".  The method is the region-based mode of
MultiDiffusion (Bar-Tal et al., "MultiDiffusion: Fusing Diffusion Paths for Controlled Image Generation", ICML 2023, section 4.2):
every step runs one UNet pass per region, each with its own context, and every latent element takes the mask-weighted average of
the regions' predictions.  It needs no retraining, and it combines with the window fusion of lib/model_zoo/panorama.py, which is
this walk with no regions (R = 0).  A region's context may be a CLIP image context, so one region can follow a reference photo
while another follows text.

API.  x_info['regions'] = Regions([Region(mask, conditioning), ...], bootstrap_steps=0, backgrounds=None) on DDIMSampler.sample /
sample_multicontext and DPMSolverSampler (same methods).
  - The call's own c_info(s) give the background prompt (region 0), the unconditional context, the types, the ratios and the
    guidance scale.
  - A Region gives a mask and a conditioning only.  The mask is fp32 [bs | 1, H, W] at latent resolution or [bs | 1, 8H, 8W] at
    pixel resolution; a pixel mask is reduced by the max over each 8x8 cell (vdb_mask_to_latent), as inpainting's.  Values lie in
    [0, 1]; soft masks are allowed.  The conditioning is one tensor shaped like the call's 'conditioning' for sample, and a list
    with one tensor per c_info (each shaped like that c_info's 'conditioning') for sample_multicontext.
  - 1 <= R <= REGIONS_MAX = 8 regions.
  - regions() below samples and decodes in one call.

Weights, per latent element p, fp32 with round-to-nearest.
  - Region weights m_r(p), r = 1..R, and their sum S = m_1 + ... + m_R in ascending r (the first term sets S).
  - The background's weight m_0 = max(0, 1 - S), the paper's rule, and the denominator D = m_0 + S: S when S >= 1, else 1 up to
    one rounding.  So D >= 1 - 2^-24 and never 0.

Merge.  Block r = 0..R is a UNet pass with context r (block 0: the background).  With j over the n(p) windows covering p in
ascending window index (one window, the canvas, when x_info['windows'] is absent) and r ascending inside each window:
    e(p) = sum_j sum_r m_r(p) e_{j,r}(p) / (n(p) D(p))
Each product is one rounded multiply; the first sets the sum, later terms are added; one division by the rounded product n D.  A
term of weight exactly 0 is skipped, not multiplied: a hard mask (m_r = 1, the others 0) selects region r's eps bit for bit, and
all-zero region masks select the background's.  As the window merge, the gather form keeps the running sum in the output between
the launches of a chunked merge (no atomics), so merging in chunks equals one merge bit for bit, and the graph path equals the
eager path.

Why averaging eps is the paper's form.  The paper averages the per-region x_{t-1} with the mask weights.  DDIM's update is
x' = a x + b eps; with binary masks m_r x_r = m_r x even under bootstrapping (below), so sum_r m_r (a x_r + b e_r) / D =
a x + b e: averaging eps and running the unchanged update on the canvas is the same step.  By linearity the same holds for
DPM-Solver++'s data predictions, and the img2img start, the inpainting blend and the DPM-Solver++ history ring run unchanged.  With
soft masks and bootstrapping the per-region inputs differ where 0 < m_r < 1, and the mask-weighted eps average is the definition.

CFG layout.  A chunk's batch is [u blocks; c blocks]; within a block, row j bs + b is window first + j of image b.
  - Without bootstrapping the unconditional half is one block, region 0's context on the plain latent, averaged over windows as a
    panorama's (vdb_region_merge_f32 at R = 0, halves = 1).  The c blocks go through vdb_region_merge_f32 at R.
  - With bootstrapping each region's input differs from the canvas, so each block has its own unconditional row (R + 1 u blocks)
    and both halves go through the weighted merge.  Then e_u + s (e_c - e_u) = sum_r m_r (u_r + s (c_r - u_r)) / D, the paper's
    per-region guided eps.

Bootstrapping (paper section 4.2).  For the first bootstrap_steps steps walked, region r >= 1 reads m_r x + (1 - m_r) (a bg + b z)
in place of x, with the exact selects of the inpainting blend at m in {0, 1}: the region is denoised against a plain background,
which pins its object inside the mask.
  - a = sqrt(ac_t) and b = sqrt(1 - ac_t) are the noise level of the latent entering the step (DDIM's ddim_alphas; DPM-Solver++
    walks the same grid).  They come from a device table row {on, a, b, 0} at the step counter (step_rows), which also holds the
    on/off flag, so one captured graph serves every step.
  - bg is a per-channel constant latent: a row of `backgrounds` (fp32 [nb, C]).  Region r of image b takes row
    floor(w nb / 2^32) of the Philox4x32-10 word w at counter (r bs + b, step, "rgns", 1).  color_backgrounds() makes such rows.
  - z is the canvas element's normal at counter (element quad, step, "rgns", 0), by the Box-Muller of the inpainting blend.  It is
    keyed per canvas element, so overlapping windows and all regions see the same z, as in the paper's code.
  - The 64-bit key is drawn from torch's CPU generator only when bootstrapping is on, after every refusal.

Step.  Inside the sampler's step, for each chunk of max(1, WINDOWS_PER_CHUNK // (R + 1)) windows (so a UNet call holds about as
many items as a panorama chunk): vdb_region_gather_f32 (canvas -> the chunk's batch, every block in one launch), the UNet on the
batch with the region contexts ([u...; c_0...; c_R...], each row repeated per window, in persistent buffers of their own), and the
merges into a persistent canvas eps [e_u; e_c].  The walk's state (RegionState: the layout tables, the masks, the step rows,
backgrounds and key while bootstrapping, the chunk batch and the canvas eps) is refilled in place, so a cached step graph replays
on new prompts and masks.

Refusals, before any device work.  ValueError: x_info['regions'] not a Regions; a text latent; a mask or conditioning of the wrong
type or shape; mask values outside [0, 1] or NaN; R outside [1, 8]; bootstrap_steps outside [0, the walk's grid points];
bootstrapping without backgrounds, or backgrounds not [nb >= 1, C]; x_info['windows'] not a panorama.Windows or a layout panorama
refuses.
NotImplementedError: prompt_edit, sampling from an inversion, PLMSSampler and the single-step p_sample_ddim.  The img2img start,
inpaint_mask (outpainting with regions) and single or dual contexts combine unchanged.  Without 'regions' nothing changes: the same
launches, the same bits, the same graph key.

Measured with tools/regions_bench.py on one NVIDIA H100 80GB HBM3 at a 700 W power limit, config 2's shape (bs 4, 512x512, CFG 7.5,
VAE decode included), vertical band masks, bootstrapping over the first 20 % of the steps, best of 5: DDIM 50 takes 1140 / 1469 /
2131 ms per call with 1 / 2 / 4 regions (1477 / 2136 / 3632 with bootstrapping) against config 2's 783 ms; DPM-Solver++ 2M 20
takes 491 / 622 / 880 ms (621 / 876 / 1486).  A UNet item costs within 8 % of config 2's; the graph path equals the eager path bit
for bit; one step's gather and merge take 0.011 ms.  A 512x2048 panorama at stride 16 with 2 regions takes 5005 ms (DDIM 50) and
2086 ms (DPM-Solver++ 2M 20); 2 windows per UNet call run 96.9 ms per step at a 241 MB sampling peak, 1 window 112.7 ms, 4
windows 93.9 ms at 520 MB.
"""
import numpy as np
import torch

from .ddim import SamplerMode, buffers_key, refuse
from .diffusion_utils import to_numpy
from .panorama import LayoutTables, Windows, layout

REGIONS_MAX = 8


def _ops():
    from vdb200 import ops
    return ops


class Region(object):
    """One region: a mask (fp32 [bs | 1, H, W] or [bs | 1, 8H, 8W], values in [0, 1]) and its conditioning (a tensor for sample,
    a list with one tensor per c_info for sample_multicontext)."""

    def __init__(self, mask, conditioning):
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.float32:
            raise ValueError(f"Region: mask must be an fp32 tensor, got {getattr(mask, 'dtype', type(mask).__name__)}")
        conds = list(conditioning) if isinstance(conditioning, (list, tuple)) else [conditioning]
        if not conds or not all(isinstance(c, torch.Tensor) for c in conds):
            raise ValueError("Region: conditioning must be a tensor, or a list of tensors (one per c_info)")
        self.mask, self.conds = mask, conds


class Regions(object):
    """x_info['regions']: 1..REGIONS_MAX Region, the steps to bootstrap and the backgrounds fp32 [nb, C] they draw from."""

    def __init__(self, regions, bootstrap_steps=0, backgrounds=None):
        regions = list(regions)
        if not 1 <= len(regions) <= REGIONS_MAX:
            raise ValueError(f"Regions: need 1 to {REGIONS_MAX} regions, got {len(regions)}")
        if not all(isinstance(r, Region) for r in regions):
            raise ValueError("Regions: every entry must be a Region")
        if not isinstance(bootstrap_steps, (int, np.integer)) or isinstance(bootstrap_steps, bool) or bootstrap_steps < 0:
            raise ValueError(f"Regions: bootstrap_steps must be an integer >= 0, got {bootstrap_steps!r}")
        if bootstrap_steps and backgrounds is None:
            raise ValueError("Regions: bootstrapping needs backgrounds (fp32 [nb, C]; see color_backgrounds)")
        if backgrounds is not None and (not isinstance(backgrounds, torch.Tensor) or backgrounds.dim() != 2 or
                                        backgrounds.shape[0] < 1 or not torch.isfinite(backgrounds.float()).all()):
            raise ValueError("Regions: backgrounds must be a finite tensor [nb >= 1, C]")
        self.regions, self.bootstrap_steps = regions, int(bootstrap_steps)
        self.backgrounds = backgrounds

    def __len__(self):
        return len(self.regions)


def weights(masks):
    """(m_0, D) of region masks [R, ...] in fp32 with the kernels' order and rounding (numpy)."""
    m = np.asarray(masks, dtype=np.float32)
    S = m[0].copy()
    for r in range(1, m.shape[0]):
        S = (S + m[r]).astype(np.float32)
    m0 = np.maximum(np.float32(0), (np.float32(1) - S).astype(np.float32))
    return m0, (m0 + S).astype(np.float32)


def step_rows(alphas, total, bootstrap_steps):
    """fp32 [total, 4] rows {on, sqrt(a), sqrt(1 - a), 0} indexed by the grid index i, a = the cumulative alpha of grid point i
    (fp64 -> fp32); on = 1 for the first bootstrap_steps steps walked (i = total - 1 down)."""
    a = to_numpy(alphas, np.float64)[:total]
    t = np.zeros((total, 4), dtype=np.float32)
    t[:, 0] = np.arange(total) >= total - bootstrap_steps
    t[:, 1], t[:, 2] = np.sqrt(a), np.sqrt(1.0 - a)
    return t


def latent_masks(regs, bs, H, W, device):
    """The regions' masks as one fp32 device tensor [R, bs, H, W] (pixel masks reduced, batch-1 masks broadcast)."""
    out = torch.empty(len(regs.regions), bs, H, W, dtype=torch.float32, device=device)
    for r, reg in enumerate(regs.regions):
        m = reg.mask.to(device=device, dtype=torch.float32).contiguous()
        if m.shape[-1] != W:
            m = _ops().mask_to_latent(m.unsqueeze(1)).squeeze(1)
        out[r].copy_(m.expand(bs, H, W))
    return out


class RegionState(LayoutTables):
    """The device side of a region walk, persistent across calls so a captured step graph replays: the layout tables, the masks
    [R, bs, H, W] (R >= 1), the step rows, the backgrounds and the key (while bootstrapping: nb > 0), the chunk batch and the
    canvas eps [e_u; e_c].  What the walk does not use is None."""

    def __init__(self, key, lay, per, bs, cfg, C, R, ub, nb, device):
        super().__init__(lay, device)
        self.key = key
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=device)
        self.masks = z(R, bs, lay.H, lay.W) if R else None
        self.rows, self.seed, self.bg = (z(1000, 4), z(1, dtype=torch.int64), z(nb, C)) if nb else (None, None, None)
        self.xw = z((ub + R + 1) * min(per, lay.nwin) * bs, lay.h, lay.w, C)
        self.eps = z((2 if cfg else 1) * bs, lay.H, lay.W, C)

    def buffers(self):
        return (self.tables, self.masks, self.rows, self.seed, self.bg, self.xw, self.eps)


class RegionPrompts(SamplerMode):
    """x_info['regions'] in the sampler's walk: the mask-weighted eps of the regions in place of the UNet call on the canvas.  With
    x_info['windows'] alone it is a panorama's window fusion: the walk with no regions (R = 0)."""

    def __init__(self, sampler, x_info, shape, c_infos):
        """The host-side refusals of a region or panorama call, before any device work."""
        regs, win = x_info.get('regions', None), x_info.get('windows', None)
        who = 'windows' if regs is None else 'regions'
        if regs is None:
            _check_windows(win)
        elif not isinstance(regs, Regions):
            raise ValueError(f"x_info['regions'] must be a regions.Regions, got {type(regs).__name__}")
        refuse(who, x_info, c_infos)
        if len(shape) != 4:
            raise ValueError(f"{who} need an image latent [bs, C, H, W], got shape {list(shape)} (a text latent?)")
        bs, C, H, W = shape
        self.regions = [] if regs is None else regs.regions
        for r, reg in enumerate(self.regions, 1):
            m = reg.mask
            if m.dim() != 3 or m.shape[0] not in (1, bs) or tuple(m.shape[1:]) not in ((H, W), (8 * H, 8 * W)):
                raise ValueError(f"region {r}: mask expected [{bs} or 1, {H}, {W}] (latent) or [{bs} or 1, {8 * H}, {8 * W}] "
                                 f"(pixel), got {tuple(m.shape)}")
            if not bool(((m >= 0) & (m <= 1)).all()):
                raise ValueError(f"region {r}: mask values must lie in [0, 1] (no NaN)")
            if len(reg.conds) != len(c_infos):
                raise ValueError(f"region {r}: {len(reg.conds)} conditioning tensors for {len(c_infos)} contexts")
            for i, (c, ci) in enumerate(zip(reg.conds, c_infos)):
                if tuple(c.shape) != tuple(ci['conditioning'].shape):
                    raise ValueError(f"region {r}: conditioning {i} expected {tuple(ci['conditioning'].shape)} (as the call's), "
                                     f"got {tuple(c.shape)}")
        if regs is not None:
            steps = len(sampler.ddim_timesteps)
            if regs.bootstrap_steps > steps:
                raise ValueError(f"Regions: bootstrap_steps must lie in [0, {steps}] (the walk's grid points), "
                                 f"got {regs.bootstrap_steps}")
            if regs.backgrounds is not None and regs.backgrounds.shape[1] != C:
                raise ValueError(f"Regions: backgrounds expected [nb, {C}], got {tuple(regs.backgrounds.shape)}")
        if win is None:
            side = max(H, W, 8)
            win = Windows(side, side)
        else:
            _check_windows(win)
        self.regs, self.R, self.boot = regs, len(self.regions), regs is not None and regs.bootstrap_steps > 0
        self.lay = layout(win, H, W)
        from . import panorama
        self.per = max(1, panorama.WINDOWS_PER_CHUNK // (self.R + 1))
        self.chunks = self.lay.chunks(self.per)

    def start(self, sampler, x_info, shape, dtype, device):
        # the Philox key, from torch's CPU generator: drawn only when bootstrapping, after every mode's refusals
        self.seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64) if self.boot else None
        return None

    def prepare(self, sampler, run):
        """Refill the RegionState in place and the region contexts, which become the contexts whose K / V^T the step reads."""
        lay, per, R, regs = self.lay, self.per, self.R, self.regs
        self.ub = (R + 1 if self.boot else 1) if run.cfg else 0
        nb = regs.backgrounds.shape[0] if self.boot else 0
        key = lay.key() + (per, run.bs, run.cfg, run.C, R, self.ub, nb)
        st = run.walk.get('regions')
        if st is None or st.key != key:
            st = run.walk['regions'] = RegionState(key, lay, per, run.bs, run.cfg, run.C, R, self.ub, nb, run.device)
        if R:
            st.masks.copy_(latent_masks(regs, run.bs, lay.H, lay.W, run.device))
        if self.boot:
            st.rows[:run.total].copy_(torch.from_numpy(step_rows(sampler.ddim_alphas, run.total, regs.bootstrap_steps)))
            st.bg.copy_(regs.backgrounds.to(device=run.device, dtype=torch.float32))
            st.seed.copy_(self.seed)
        self.st = st
        self.ctxs = {k: region_contexts(sampler, run, self.regions, k, self.ub) for k in sorted({k for _, k in self.chunks})}
        run.kv_types = [ct for _ in self.ctxs for ct in run.c_types]
        run.kv_ctxs = [c for k in self.ctxs for c in self.ctxs[k]]
        return ('regions', lay.key(), per, R, self.ub, nb) + buffers_key(*st.buffers())

    def eps(self, sampler, run):
        """gather -> UNet -> merge per chunk of windows, into the canvas eps [e_u; e_c]"""
        ops, st, lay, bs, R, ub = _ops(), self.st, self.lay, run.bs, self.R, self.ub
        boot = dict(rows=st.rows, step_idx=run.walk['idx'], seed=st.seed, bg=st.bg) if self.boot else {}
        t_emb = ops.timestep_embedding(run.walk['ts'], run.mch, step_idx=run.walk['idx'], batch=st.xw.shape[0])
        for first, k in self.chunks:
            rows = k * bs
            xw = st.xw[:(ub + R + 1) * rows]
            ops.region_gather(run.x, st.oy, st.ox, lay.h, lay.w, first, k, R, ub, out=xw, masks=st.masks, **boot)
            e = sampler.model.eps_nhwc(xw, run.x_type, t_emb[:xw.shape[0]], run.c_types, self.ctxs[k], run.ratios, run.time_from)
            tabs = (st.oy, st.ox, st.cover_y, st.cover_x, first, k)
            if ub == 1 and R:   # one u block on the plain latent: the window average (R = 0); the c blocks: the weighted merge
                ops.region_merge(e[:rows], *tabs, 0, None, st.eps[:bs], halves=1)
                ops.region_merge(e[rows:], *tabs, R, st.masks, st.eps[bs:], halves=1)
            else:
                ops.region_merge(e, *tabs, R, st.masks, st.eps, halves=2 if ub else 1)
        return st.eps


def _check_windows(win):
    if not isinstance(win, Windows):
        raise ValueError(f"x_info['windows'] must be a panorama.Windows, got {type(win).__name__}")


def region_contexts(sampler, run, regions, k, ub):
    """The contexts of a chunk of k windows, one per c_info, in persistent buffers of their own: blocks [u x ub; c_0; c_1 ..
    c_R] (c_1 .. c_R from the Region list `regions`, none for a panorama), each block's bs rows repeated k times (row j bs + b is
    image b)."""
    from .attention import PaddedContext
    ctxs = []
    for i, ci in enumerate(run.c_infos):
        c0 = ci['conditioning']
        blocks = [ci['unconditional_conditioning']] * ub + [c0] + [reg.conds[i] for reg in regions]
        c = torch.cat([b.to(device=c0.device, dtype=c0.dtype).repeat(k, 1, 1) for b in blocks])
        ctxs.append(PaddedContext(sampler._ctx_buffer((('regions', k), i), c), c.shape[1]))
    return ctxs


@torch.no_grad()
def color_backgrounds(net, colors):
    """Backgrounds for bootstrapping: each RGB colour in [0, 1] (a [nb, 3] sequence) as a uniform 64x64 image, encoded to the
    posterior mode and averaged per channel -> fp32 [nb, 4] on the model's device."""
    col = torch.as_tensor(np.asarray(colors, dtype=np.float32)).reshape(-1, 3)
    n = col.shape[0]
    img = col[:, :, None, None].expand(n, 3, 64, 64).contiguous().to(net.device)
    z = net.vae_encode(img * 2 - 1, 'image', noise=torch.zeros(n, 4, 8, 8))
    return z.double().cpu().mean(dim=(2, 3)).float().to(net.device)


@torch.no_grad()
def regions(net, sampler, c_info, regions, height=512, width=512, steps=50, n=1, windows=None, x_info=None, **kw):
    """Sample n images of height x width pixels with region prompts and decode them -> [n, 3, height, width] in [0, 1].  c_info:
    the background's context dict, or a list for sample_multicontext; regions: a Regions; windows: an optional panorama.Windows
    for a wide canvas; x_info: further x_info entries ('xt', 'x0' and 'x0_forward_timesteps', 'inpaint_mask').  Other keywords go
    to the sampler."""
    if height % 8 or width % 8:
        raise ValueError(f"height and width must be multiples of 8, got {height} x {width}")
    xi = dict(x_info or {}, type='image', regions=regions)
    if windows is not None:
        xi['windows'] = windows
    shape = [n, 4, height // 8, width // 8]
    kw.setdefault('verbose', False)
    if isinstance(c_info, (list, tuple)):
        z, _ = sampler.sample_multicontext(steps=steps, shape=shape, x_info=xi, c_info_list=list(c_info), **kw)
    else:
        z, _ = sampler.sample(steps=steps, shape=shape, x_info=xi, c_info=c_info, **kw)
    return net.vae_decode(z, 'image')
