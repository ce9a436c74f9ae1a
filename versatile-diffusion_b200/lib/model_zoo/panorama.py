"""Panoramas and large canvases — MultiDiffusion window fusion inside the captured DDIM / DPM-Solver++ step graph.

The reference has no panorama mode; this is an addition, and its semantics are specified here.  The model was trained on 64x64
latents: sampled whole at 64x256 it repeats objects and loses the composition.  MultiDiffusion (Bar-Tal et al., "MultiDiffusion:
Fusing Diffusion Paths for Controlled Image Generation", ICML 2023) needs no retraining: each step denoises overlapping windows of
the canvas, and every canvas element takes the average of the windows that cover it.

API.  x_info['windows'] = Windows(size=64, stride=8, circular=False) on DDIMSampler.sample / sample_multicontext and
DPMSolverSampler (same methods), with any context set-up (text, image, dual, multi), the img2img start (x0 +
x0_forward_timesteps) and inpaint_mask (lib/model_zoo/inpaint.py; a mask on a wide canvas outpaints a photo into a panorama).
panorama() below samples and decodes in one call.

Layout, computed once on the host (layout()) and uploaded as small int32 device tables.
  - The window side along each axis is min(size, canvas side): h x w.
  - Origins along an axis are 0, s, 2s, ..., plus one final window flush with the far edge when the stride does not land
    there, so every element is covered.  circular=True wraps along W for 360-degree panoramas: origins 0, s, ..., W - s, windows
    read columns (origin + j) mod W across the seam, and W % stride must be 0.  H never wraps.
  - Window g = iy * nx + ix has origin (oy[iy], ox[ix]).

Equivalence.  The paper averages the per-window x_{t-1}.  Every update here is linear in eps: DDIM's x' = a x + b eps (pointwise,
the same a and b for every window), the CFG mix, and DPM-Solver++'s data predictions.  So averaging per-window x_{t-1} equals
averaging the per-window eps into a canvas eps and running the unchanged update on the whole canvas.  Under CFG the unconditional
and conditional halves are averaged separately, then mixed by vdb_ddim_cfg_step / vdb_dpmpp_cfg_step.

Step.  A panorama is the region walk of lib/model_zoo/regions.py with no regions (R = 0).  Inside the sampler's step, the UNet
call on the canvas becomes, for each chunk of at most WINDOWS_PER_CHUNK windows in window order: vdb_region_gather_f32 at R = 0
(canvas -> [u rows of the chunk's windows; c rows], exact copies), the UNet on that batch with window contexts (each context row
repeated per window, in persistent buffers of their own), and vdb_region_merge_f32 at R = 0 into a persistent canvas eps
[e_u; e_c].  Everything after it is untouched: the update, the inpainting blend, the DPM-Solver++ history ring (which holds the
canvas).

Merge.  Uniform weights, as in the paper (at R = 0 every weight of the region merge is 1 and its D is 1, exactly).  Each canvas element is the fp32 sum of the eps of its covering windows, taken in
ascending window index, divided by the integer count: the first window sets the sum, each later one is added with
round-to-nearest, and the division is one round-to-nearest.  Each output element loops over its covering windows (gather form):
no atomics, so the result is bit-reproducible and the graph path equals the eager path.  Merges over consecutive chunks make the
same operations in the same order as one merge over all windows; the UNet's own reductions are split by batch size, so another
chunk size changes the last bits of each window's eps, not the merge.
With a single covering window the result is that window's eps bit for bit; so a window equal to the canvas gives the unwindowed
sampler's result bit for bit.

Refusals, before any device work.  ValueError: a text latent ([n, 768]), x_info['windows'] not a Windows, size below 8, stride
not in [1, size], circular with W % stride != 0.  NotImplementedError: prompt_edit (its item tables index prompts, not windows),
sampling from an inversion, PLMSSampler, and the single-step p_sample_ddim.  Without 'windows' nothing changes: the same
launches, the same bits, the same graph key.

Known limit.  The VAE decode is not tiled: its mid-block attention materialises an N x N score matrix per image, 512 MB in bf16 at
a 64x256 latent, and it grows quadratically with wider canvases.
"""
import numpy as np
import torch


# Windows per UNet call.  A chunk's UNet batch is 2 * WINDOWS_PER_CHUNK * n under CFG; larger chunks amortise the per-call launch
# overhead, smaller ones bound the activation memory on large canvases.  tools/panorama_bench.py, DPM-Solver++ 20 at 512x2048 and
# stride 8 (25 windows), one NVIDIA H100 80GB HBM3 at a 700 W power limit: chunks of 1 / 4 / 8 / 13 / 25 windows take 149.3 /
# 97.3 / 96.7 / 94.8 / 97.1 ms per step, with a sampling peak of 64 / 242 / 478 / 933 / 1717 MB above what was allocated before.
# 8 is within 2 % of the fastest at half the memory of 13.
WINDOWS_PER_CHUNK = 8


class Windows(object):
    """A MultiDiffusion window layout request: square windows of `size` latent elements (clamped to the canvas), `stride` apart,
    optionally wrapping along W."""

    def __init__(self, size=64, stride=8, circular=False):
        if not isinstance(size, (int, np.integer)) or size < 8:
            raise ValueError(f"Windows: size must be an integer >= 8 (latent elements), got {size!r}")
        if not isinstance(stride, (int, np.integer)) or not 1 <= stride <= size:
            raise ValueError(f"Windows: stride must be an integer in [1, size={size}], got {stride!r}")
        self.size, self.stride, self.circular = int(size), int(stride), bool(circular)

    def __repr__(self):
        return f"Windows(size={self.size}, stride={self.stride}, circular={self.circular})"


def axis_origins(L, size, stride, circular=False):
    """(window side, origins) along an axis of L elements."""
    side = min(size, L)
    if circular:
        return side, list(range(0, L, stride))
    origins = list(range(0, L - side + 1, stride))
    if origins[-1] != L - side:
        origins.append(L - side)
    return side, origins


def axis_cover(L, side, origins, circular=False):
    """int32 [L, 4] {a0, a1, b0, b1}: the windows covering position p are [a0, a1) then [b0, b1), ascending.  A circular axis
    covers a cyclic run of windows, which in ascending order is at most two runs: [0, a1) and [b0, n)."""
    n = len(origins)
    o = np.asarray(origins)
    # one run is stored as {lo, hi, hi, hi}
    out = np.zeros((L, 4), dtype=np.int32)
    for p in range(L):
        d = (p - o) % L if circular else p - o
        idx = np.nonzero((d >= 0) & (d < side))[0]
        breaks = np.nonzero(np.diff(idx) != 1)[0]
        if len(breaks) == 0:
            out[p] = (idx[0], idx[-1] + 1, idx[-1] + 1, idx[-1] + 1)
        else:
            assert circular and len(breaks) == 1 and idx[0] == 0 and idx[-1] == n - 1, (p, idx)
            out[p] = (0, idx[breaks[0]] + 1, idx[breaks[0] + 1], n)
    return out


class Layout(object):
    """The host tables of a window layout on an H x W canvas."""

    def __init__(self, windows, H, W):
        if windows.circular and W % windows.stride:
            raise ValueError(f"Windows: circular needs the canvas width {W} to be a multiple of the stride {windows.stride}")
        self.windows, self.H, self.W = windows, H, W
        self.h, oy = axis_origins(H, windows.size, windows.stride)
        self.w, ox = axis_origins(W, windows.size, windows.stride, windows.circular)
        self.oy, self.ox = np.asarray(oy, dtype=np.int32), np.asarray(ox, dtype=np.int32)
        self.ny, self.nx = len(oy), len(ox)
        self.nwin = self.ny * self.nx
        self.cover_y = np.ascontiguousarray(axis_cover(H, self.h, oy)[:, :2])     # H never wraps: one run {lo, hi}
        self.cover_x = axis_cover(W, self.w, ox, windows.circular)

    def key(self):
        w = self.windows
        return (self.H, self.W, w.size, w.stride, w.circular)

    def counts(self):
        """int [H, W]: how many windows cover each element."""
        cy = self.cover_y[:, 1] - self.cover_y[:, 0]
        cx = (self.cover_x[:, 1] - self.cover_x[:, 0]) + (self.cover_x[:, 3] - self.cover_x[:, 2])
        return cy[:, None] * cx[None, :]

    def chunks(self, per=None):
        """[(first, k)]: consecutive ranges of at most `per` (default WINDOWS_PER_CHUNK) windows, in window order."""
        per = WINDOWS_PER_CHUNK if per is None else per
        return [(f, min(per, self.nwin - f)) for f in range(0, self.nwin, per)]

    def table(self):
        """All tables in one int32 array: cover_x [W, 4] first (its rows are read as int4), then cover_y [H, 2], oy, ox ->
        (array, {name: (offset, length)})."""
        parts = [("cover_x", self.cover_x.ravel()), ("cover_y", self.cover_y.ravel()), ("oy", self.oy), ("ox", self.ox)]
        offs, o = {}, 0
        for name, a in parts:
            offs[name] = (o, a.size)
            o += a.size
        return np.concatenate([a for _, a in parts]).astype(np.int32), offs


def layout(windows, H, W):
    return Layout(windows, H, W)


class LayoutTables(object):
    """A layout's int32 tables on the device, in one buffer (`tables`) read through the views cover_x, cover_y, oy and ox.  They
    depend on the layout's key alone, so state kept under that key never needs them refilled."""

    def __init__(self, lay, device):
        tab, offs = lay.table()
        self.tables = torch.from_numpy(tab).to(device)
        for name, (o, n) in offs.items():
            setattr(self, name, self.tables[o:o + n])


@torch.no_grad()
def panorama(net, sampler, c_info, height=512, width=2048, steps=50, n=1, windows=None, x_info=None, **kw):
    """Sample n images of height x width pixels with window fusion and decode them -> [n, 3, height, width] in [0, 1].  c_info:
    one context dict, or a list for sample_multicontext.  windows: a Windows (default Windows()); x_info: further x_info
    entries ('xt', 'x0' and 'x0_forward_timesteps', 'inpaint_mask').  Other keywords go to the sampler."""
    if height % 8 or width % 8:
        raise ValueError(f"height and width must be multiples of 8, got {height} x {width}")
    xi = dict(x_info or {}, type='image', windows=Windows() if windows is None else windows)
    shape = [n, 4, height // 8, width // 8]
    kw.setdefault('verbose', False)
    if isinstance(c_info, (list, tuple)):
        z, _ = sampler.sample_multicontext(steps=steps, shape=shape, x_info=xi, c_info_list=list(c_info), **kw)
    else:
        z, _ = sampler.sample(steps=steps, shape=shape, x_info=xi, c_info=c_info, **kw)
    return net.vae_decode(z, 'image')
