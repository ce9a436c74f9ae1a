"""Region prompts on the GPU (lib/model_zoo/regions.py): vdb_region_gather_f32 bitwise against a numpy fp32 restatement (layouts
including circular ones, bs, R, the u-block layouts, the bootstrap flag on and off, soft and hard masks), its Philox path equal to
the noise path fed from vdb_region_noise_f32; vdb_region_merge_f32 bitwise against its fp32 restatement in the same order and
within 1e-6 of fp64, chunked merges equal to one merge, hard and all-zero masks selecting exactly; the region DDIM and
DPM-Solver++ walks on the mini UNet against the oracle (oracle/regions_oracle.py); graph equal to eager, and a cached graph
replayed on new prompts and masks."""
import numpy as np
import pytest
import torch

from oracle import regions_oracle as G
from test_panorama_gpu import merge_restated as window_average_restated
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


def _tables(lay):
    from lib.model_zoo.panorama import LayoutTables
    return LayoutTables(lay, DEV)


def _masks(kind, R, bs, H, W, seed):
    """fp32 [R, bs, H, W]: 'soft' uniform values with exact 0 / 1 patches, 'hard' a label map (one region or the background per
    element), 'zero' all zeros"""
    g = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((R, bs, H, W), F32)
    if kind == "hard":
        lab = g.integers(0, R + 1, size=(bs, H, W))
        return np.stack([(lab == r) for r in range(1, R + 1)]).astype(F32)
    m = g.random((R, bs, H, W)).astype(F32)
    m[:, :, :3, :3] = 0.0
    m[:, :, -3:, -3:] = 1.0
    return m


LAYOUTS = [(16, 24, 64, 8, False), (16, 40, 16, 8, False), (24, 20, 16, 7, False), (16, 40, 16, 8, True), (40, 40, 16, 5, True)]


def gather_restated(x, wins, h, w, first, k, R, ub, masks, on, a, b, bg, picks, z):
    """vdb_region_gather_f32 in numpy fp32: blocks [u x ub; c_0 .. c_R], each an exact copy, or m x + (1 - m)(a bg + b z) for
    region r >= 1 while the flag is on"""
    bs, H, W, C = x.shape
    blocks = ([0] if ub == 1 else list(range(ub))) + list(range(R + 1))
    a, b = F32(a), F32(b)
    out = []
    for r in blocks:
        xr = x
        if on and r > 0:
            m = masks[r - 1][..., None]
            k_ = (a * bg[picks[r - 1]][:, None, None, :]).astype(F32) + (b * z).astype(F32)
            blend = ((m * x).astype(F32) + ((F32(1) - m).astype(F32) * k_).astype(F32)).astype(F32)
            xr = np.where(m == 1, x, np.where(m == 0, k_, blend)).astype(F32)
        for g in range(first, first + k):
            oy, ox = wins[g]
            out.append(xr[:, oy:oy + h][:, :, (ox + np.arange(w)) % W])
    return np.concatenate(out)


@pytest.mark.parametrize("H,W,size,stride,circular", LAYOUTS)
@pytest.mark.parametrize("bs,C,R", [(1, 4, 1), (3, 4, 3), (2, 3, 2), (1, 4, 8)])
def test_gather_bitwise_against_numpy(H, W, size, stride, circular, bs, C, R):
    from lib.model_zoo.panorama import Windows, layout
    from vdb200 import ops
    lay = layout(Windows(size, stride, circular), H, W)
    ws = _tables(lay)
    g = np.random.default_rng(H * W + bs * 7 + R)
    x = g.standard_normal((bs, H, W, C)).astype(F32)
    bg = g.standard_normal((5, C)).astype(F32)
    seed = torch.tensor([int(g.integers(-2 ** 62, 2 ** 62))], dtype=torch.int64, device=DEV)
    wins = [(int(oy), int(ox)) for oy in lay.oy for ox in lay.ox]
    rows = np.array([[0, 0.9, 0.4, 0], [1, 0.8, 0.6, 0], [1, 0.5, 0.75, 0]], F32)
    for kind in ("soft", "hard"):
        masks = _masks(kind, R, bs, H, W, R + bs)
        dm, dx, drows, dbg = _dev(masks), _dev(x), _dev(rows), _dev(bg)
        for step in (0, 1, 2):
            z, picks = ops.region_noise(seed, _idx(step), x.size, R, bs, bg.shape[0])
            z, picks = z.view(bs, H, W, C), picks.cpu().numpy()
            assert picks.min() >= 0 and picks.max() < bg.shape[0]
            for ub in (0, 1, R + 1):
                for first, k in lay.chunks(2) + [(0, lay.nwin)]:
                    shape = ((ub + R + 1) * k * bs, lay.h, lay.w, C)
                    out = torch.full(shape, float("nan"), device=DEV)
                    ops.region_gather(dx, ws.oy, ws.ox, lay.h, lay.w, first, k, R, ub, out=out, masks=dm, rows=drows,
                                      step_idx=_idx(step), seed=seed, bg=dbg)
                    want = gather_restated(x, wins, lay.h, lay.w, first, k, R, ub, masks, rows[step, 0] != 0, rows[step, 1],
                                           rows[step, 2], bg, picks, z.cpu().numpy())
                    assert np.array_equal(out.cpu().numpy(), want), (kind, step, ub, first, k)
                    fed = torch.full(shape, float("nan"), device=DEV)
                    ops.region_gather(dx, ws.oy, ws.ox, lay.h, lay.w, first, k, R, ub, out=fed, masks=dm, rows=drows,
                                      step_idx=_idx(step), seed=seed, bg=dbg, noise=z)
                    assert torch.equal(fed, out), "the Philox path equals the noise path"
                    if step == 0:       # flag off, and no rows at all: exact copies of the windows in every block
                        plain = torch.full(shape, float("nan"), device=DEV)
                        ops.region_gather(dx, ws.oy, ws.ox, lay.h, lay.w, first, k, R, ub, out=plain)
                        assert torch.equal(plain, out)
                        win = np.concatenate([x[:, oy:oy + lay.h][:, :, (ox + np.arange(lay.w)) % W]
                                              for oy, ox in wins[first:first + k]])
                        assert np.array_equal(plain.cpu().numpy().reshape(ub + R + 1, *win.shape),
                                              np.broadcast_to(win, (ub + R + 1,) + win.shape))


def merge_restated(eps, wins, lay, bs, halves, R, masks, C):
    """vdb_region_merge_f32 in numpy fp32, per element: windows ascending, regions ascending inside each, zero weights skipped,
    first term sets, later ones add (rounded), one division by the rounded n D"""
    from lib.model_zoo.regions import weights
    H, W, h, w = lay.H, lay.W, lay.h, lay.w
    n = len(wins)
    e = eps.reshape(halves, R + 1, n, bs, h, w, C)
    m0, Dn = weights(masks)
    m = np.concatenate([m0[None], masks])
    acc = np.zeros((halves, bs, H, W, C), F32)
    seen = np.zeros((bs, H, W), bool)
    cnt = np.zeros((H, W), np.int64)
    for g, (oy, ox) in enumerate(wins):
        cols = (ox + np.arange(w)) % W
        for r in range(R + 1):
            mr = m[r][:, oy:oy + h][:, :, cols]                          # [bs, h, w]
            blk = acc[:, :, oy:oy + h][:, :, :, cols]
            term = (mr[None, :, :, :, None] * e[:, r, g]).astype(F32)
            s = seen[:, oy:oy + h][:, :, cols]
            new = np.where(s[None, ..., None], (blk + term).astype(F32), term)
            acc[:, :, oy:oy + h, cols] = np.where((mr != 0)[None, ..., None], new, blk)
            sv = seen[:, oy:oy + h]
            sv[:, :, cols] = s | (mr != 0)
            seen[:, oy:oy + h] = sv
        cnt[oy:oy + h, cols] += 1
    dn = (cnt[None].astype(F32) * Dn).astype(F32)
    return (acc / dn[None, ..., None]).astype(F32).reshape(halves * bs, H, W, C), m, Dn, cnt


@pytest.mark.parametrize("H,W,size,stride,circular", LAYOUTS)
@pytest.mark.parametrize("bs,halves,C,R", [(1, 2, 4, 2), (2, 1, 4, 1), (3, 2, 4, 3), (2, 2, 5, 2), (1, 1, 4, 8)])
def test_merge_bitwise_against_numpy_and_fp64(H, W, size, stride, circular, bs, halves, C, R):
    from lib.model_zoo.panorama import Windows, layout
    from vdb200 import ops
    lay = layout(Windows(size, stride, circular), H, W)
    ws = _tables(lay)
    wins = [(int(oy), int(ox)) for oy in lay.oy for ox in lay.ox]
    n = lay.nwin
    g = np.random.default_rng(n * 31 + bs + R)
    eps = g.standard_normal((halves * (R + 1) * n * bs, lay.h, lay.w, C)).astype(F32)
    per_window = eps.reshape(halves, R + 1, n, bs, lay.h, lay.w, C)
    for kind in ("soft", "hard", "zero"):
        masks = _masks(kind, R, bs, H, W, n + R)
        dm = _dev(masks)
        want, m, Dn, cnt = merge_restated(eps, wins, lay, bs, halves, R, masks, C)
        assert np.array_equal(cnt, lay.counts())
        outs = []
        for per in (n, 3, 1):
            out = torch.full((halves * bs, H, W, C), float("nan"), device=DEV)
            for first, k in lay.chunks(per):
                e = np.ascontiguousarray(per_window[:, :, first:first + k]).reshape(halves * (R + 1) * k * bs, lay.h, lay.w, C)
                ops.region_merge(_dev(e), ws.oy, ws.ox, ws.cover_y, ws.cover_x, first, k, R, dm, out, halves=halves)
            outs.append(out.cpu().numpy())
        got = outs[0]
        assert np.array_equal(got, want), (kind, np.abs(got - want).max())
        for o in outs[1:]:
            assert np.array_equal(o, got), "chunked merges compute what one merge does"
        # fp64: sum_j sum_r m_r e / (n D) with the exact weights
        e64 = per_window.astype(np.float64)
        ref = np.zeros((halves, bs, H, W, C))
        for gi, (oy, ox) in enumerate(wins):
            cols = (ox + np.arange(lay.w)) % W
            for r in range(R + 1):
                ref[:, :, oy:oy + lay.h, cols] += (m[r][:, oy:oy + lay.h][:, :, cols][None, ..., None].astype(np.float64) *
                                                   e64[:, r, gi])
        S = masks.astype(np.float64).sum(0)
        ref = (ref / (cnt[None] * (np.maximum(0, 1 - S) + S))[None, ..., None]).reshape(got.shape)
        rel = np.abs(got - ref).max() / np.abs(ref).max()
        assert rel <= 1e-6, (kind, rel)
        # selection: where one weight is 1 and the rest 0 and one window covers, the selected eps bit for bit
        sel = np.argmax(m, axis=0)                                          # [bs, H, W]
        exact = (m.max(0) == 1) & ((m != 0).sum(0) == 1) & (cnt[None] == 1)
        picked = np.zeros_like(got).reshape(halves, bs, H, W, C)
        for gi, (oy, ox) in enumerate(wins):
            cols = (ox + np.arange(lay.w)) % W
            for r in range(R + 1):
                selw = sel[:, oy:oy + lay.h][:, :, cols] == r
                tmp = picked[:, :, oy:oy + lay.h][:, :, :, cols]
                tmp[:, selw] = per_window[:, r, gi][:, selw]
                picked[:, :, oy:oy + lay.h, cols] = tmp
        ex = np.broadcast_to(exact[None, ..., None], picked.shape)
        assert np.array_equal(got.reshape(picked.shape)[ex], picked[ex]), kind
        if kind == "zero":
            bg_only = np.ascontiguousarray(per_window[:, 0]).reshape(halves * n * bs, lay.h, lay.w, C)
            avg, _ = window_average_restated(bg_only, lay, wins, bs, halves, C)
            assert np.array_equal(got, avg), "all-zero masks: the background's window average bit for bit"
        if kind == "hard":
            assert exact[:, cnt == 1].all()
        print(f"[regions] merge {H}x{W} size {size} stride {stride} circular {circular} bs {bs} halves {halves} R {R} {kind}: "
              f"rel err vs fp64 {rel:.2e}")


# ---- the samplers on the mini UNet -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=7.5, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _sampler(kind, net, **kw):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return DDIMSampler(net, **kw) if kind == "ddim" else DPMSolverSampler(net, order=2, **kw)


@pytest.mark.parametrize("kind,H,W,stride,circular,multi,masked,boot,mask_kind", [
    ("ddim", 16, 24, None, False, False, False, 0, "soft"), ("ddim", 16, 24, None, False, False, False, 2, "hard"),
    ("ddim", 16, 40, 8, False, False, False, 2, "hard"), ("ddim", 16, 40, 8, True, True, False, 0, "soft"),
    ("ddim", 16, 40, 8, False, False, True, 0, "soft"), ("dpmpp", 16, 24, None, False, False, False, 2, "hard"),
    ("dpmpp", 16, 40, 8, True, False, False, 2, "soft"), ("dpmpp", 16, 40, 8, False, True, True, 2, "hard")])
def test_sampler_vs_oracle(mini, kind, H, W, stride, circular, multi, masked, boot, mask_kind):
    from lib.model_zoo import panorama
    from lib.model_zoo.regions import Region, Regions
    from vdb200 import ops
    net, sd, gi = mini
    g = torch.Generator().manual_seed(H * W + boot + multi)
    bs, C, steps, R = 1, 4, 5, 2
    xT = torch.randn(bs, C, H, W, generator=g)
    rnd = lambda L: torch.randn(bs, L, 768, generator=g) * 0.5
    if multi:
        conds, unconds = [rnd(77), rnd(257)], [rnd(77), torch.zeros(bs, 257, 768)]
        region_conds = [[rnd(77), rnd(257)] for _ in range(R)]
        oracle_kw = dict(c_types=("text", "image"), ratios=[0.7, 0.3])
        cl = [_cinfo(conds[0], unconds[0], ratio=0.7), _cinfo(conds[1], unconds[1], typ="image", ratio=0.3)]
    else:
        conds, unconds = [gi["c"][:bs]], [gi["u"][:bs]]
        region_conds = [[rnd(77)] for _ in range(R)]
        oracle_kw = {}
        cl = [_cinfo(conds[0], unconds[0])]
    masks = _masks(mask_kind, R, bs, H, W, H + W + boot)
    bgs = (torch.randn(3, C, generator=g) * 0.5) if boot else None
    regs = Regions([Region(_dev(masks[r]), [c.to(DEV) for c in region_conds[r]] if multi else region_conds[r][0].to(DEV))
                    for r in range(R)], bootstrap_steps=boot, backgrounds=None if bgs is None else bgs.to(DEV))
    x_info = {"type": "image", "xt": xT.to(DEV), "regions": regs}
    if stride is not None:
        x_info["windows"] = panorama.Windows(16, stride, circular)
    x0 = mask = None
    if masked:         # outpainting: keep a photo's latent in the middle, generate both sides
        x0 = torch.randn(1, C, H, W, generator=g) * 0.8
        mask = torch.ones(1, 1, H, W)
        mask[..., W // 2 - 6:W // 2 + 6] = 0.0
        x_info.update(x0=x0.to(DEV), inpaint_mask=mask.to(DEV))
    S = _sampler(kind, net)
    with torch.no_grad():
        kw = dict(steps=steps, shape=[bs, C, H, W], x_info=x_info, verbose=False, eta=0.)
        x, _ = S.sample_multicontext(c_info_list=cl, **kw) if multi else S.sample(c_info=cl[0], **kw)
    st = S._st
    z_fn = pick_fn = noise_fn = None
    if boot:
        seed = st["regions"].seed.clone()
        draws = lambda i: ops.region_noise(seed, _idx(i), bs * H * W * C, R, bs, bgs.shape[0])
        z_fn = lambda i: draws(i)[0].view(bs, H, W, C).permute(0, 3, 1, 2).cpu().double().numpy()
        pick_fn = lambda i: draws(i)[1].cpu().numpy()
    if masked:
        iseed = st["seed"].clone()
        noise_fn = lambda i: ops.inpaint_noise(iseed, _idx(i), bs * H * W * C).view(bs, H, W, C).permute(0, 3, 1, 2).cpu()
    ref = G.sample(sd, xT, conds, unconds, region_conds, masks.astype(np.float64), steps, size=None if stride is None else 16,
                   stride=stride, circular=circular, sampler=kind, order=2, scale=7.5, bootstrap_steps=boot,
                   backgrounds=None if bgs is None else bgs.numpy(), pick_fn=pick_fn, z_fn=z_fn, x0=x0, mask=mask,
                   noise_fn=noise_fn, model_channels=64, **oracle_kw)
    _cmp(x, ref, cos_min=0.999, tol=0.1, what=f"regions {kind} {H}x{W} stride {stride} circular {circular} "
                                                f"{'dual' if multi else 'single'} {'masked ' if masked else ''}boot {boot} "
                                                f"{mask_kind} masks vs oracle")
    if masked:
        keep = (mask == 0).expand(bs, C, H, W)
        assert torch.equal(x.cpu()[keep], x0.expand(bs, C, H, W)[keep]), "the kept region is x0 exactly"


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_graph_equals_eager_and_replays_on_new_prompts_and_masks(mini, kind):
    from lib.model_zoo import panorama
    from lib.model_zoo.regions import Region, Regions
    net, sd, gi = mini
    g = torch.Generator().manual_seed(43)
    bs, C, H, W, R = 2, 4, 16, 40, 2
    xT = torch.randn(bs, C, H, W, generator=g).to(DEV)
    c, u = gi["c"].repeat(bs, 1, 1).to(DEV), gi["u"].repeat(bs, 1, 1).to(DEV)
    bgs = (torch.randn(3, C, generator=g) * 0.5).to(DEV)

    def regs(seed, boot=2):
        gg = torch.Generator().manual_seed(seed)
        return Regions([Region(_dev(_masks("soft", 1, 1, H, W, seed + r)[0]), (torch.randn(bs, 77, 768, generator=gg) * 0.5).to(DEV))
                        for r in range(R)], bootstrap_steps=boot, backgrounds=bgs)

    def run(S, rg, windows=panorama.Windows(16, 8)):
        x_info = {"type": "image", "xt": xT.clone(), "regions": rg}
        if windows is not None:
            x_info["windows"] = windows
        torch.manual_seed(7)
        with torch.no_grad():
            return S.sample(steps=6, shape=[bs, C, H, W], x_info=x_info, c_info=_cinfo(c, u, scale=5.0), verbose=False, eta=0.)[0]

    Sg = _sampler(kind, net)
    g1 = run(Sg, regs(1))
    assert torch.equal(g1, run(_sampler(kind, net, use_cuda_graph=False), regs(1))), "graph path equals eager path"
    graph = next(iter(Sg._graphs.values()))[0]
    launches = Sg.last_step_launches
    Sg.last_step_launches = None
    g2 = run(Sg, regs(2))
    assert next(iter(Sg._graphs.values()))[0] is graph, "the second call replays the cached graph"
    assert Sg.last_step_launches is None, "without an eager step"
    assert torch.equal(g2, run(_sampler(kind, net), regs(2))), "replay on refilled prompts and masks equals a fresh sampler"
    assert not torch.equal(g2, g1) and torch.isfinite(g1).all()
    # launches per step, for the record (the UNet's own launches depend on its batch)
    S0 = _sampler(kind, net)
    run(S0, regs(3, boot=0), windows=None)
    Sp = _sampler(kind, net)
    x_info = {"type": "image", "xt": xT.clone()}
    with torch.no_grad():
        Sp.sample(steps=6, shape=[bs, C, H, W], x_info=x_info, c_info=_cinfo(c, u, scale=5.0), verbose=False, eta=0.)
    print(f"[regions] {kind} launches per step: plain {Sp.last_step_launches}, regions {S0.last_step_launches}, "
          f"regions + 4 windows + bootstrap {launches}")


def test_color_backgrounds_and_the_helper():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.regions import Region, Regions, color_backgrounds, regions
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=True)
    bg = color_backgrounds(net, [[1, 1, 1], [0.2, 0.5, 0.9]])
    assert bg.shape == (2, 4) and bg.dtype == torch.float32 and torch.isfinite(bg).all()
    assert not torch.equal(bg[0], bg[1])
    gi = golden_inputs("mini")
    m = torch.zeros(1, 128, 256, device=DEV)
    m[..., :128] = 1.0
    rg = Regions([Region(m, (gi["c"] * 0.5).to(DEV))], bootstrap_steps=2, backgrounds=bg)
    torch.manual_seed(0)
    out = regions(net, DDIMSampler(net), _cinfo(gi["c"], gi["u"]), rg, height=128, width=256, steps=5)
    assert out.shape == (1, 3, 128, 256) and torch.isfinite(out).all()
