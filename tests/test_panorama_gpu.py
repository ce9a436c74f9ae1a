"""Panoramas on the GPU (lib/model_zoo/panorama.py): vdb_region_gather_f32 at R = 0 bitwise against a numpy copy,
vdb_region_merge_f32 at R = 0 bitwise against the window average's fp32 restatement in the same order and within 1e-6 of fp64,
chunked merges equal to one merge; the
windowed DDIM and DPM-Solver++ samplers on the mini UNet against the MultiDiffusion oracle (oracle/panorama_oracle.py); the
invariants (a window equal to the canvas gives the unwindowed result bit for bit, graph equals eager, a cached graph replays on
new prompts, other chunk sizes agree); and a wide latent through the mini VAE."""
import numpy as np
import pytest
import torch

from oracle import panorama_oracle as P
from oracle import vd_oracle as O
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _tables(lay):
    from lib.model_zoo.panorama import LayoutTables
    return LayoutTables(lay, DEV)


def _crop_nhwc(x, oy, ox, h, w):
    """x [bs, H, W, C] -> the window's [bs, h, w, C], columns mod W"""
    return x[:, oy:oy + h][:, :, (ox + np.arange(w)) % x.shape[2]]


LAYOUTS = [(16, 40, 16, 8, False), (24, 20, 16, 7, False), (32, 32, 16, 8, False), (16, 40, 16, 8, True), (64, 256, 64, 8, False),
           (64, 256, 64, 16, True), (40, 40, 16, 5, True)]


@pytest.mark.parametrize("H,W,size,stride,circular", LAYOUTS)
@pytest.mark.parametrize("bs,C", [(1, 4), (3, 4), (2, 3)])
def test_gather_with_no_regions_bitwise(H, W, size, stride, circular, bs, C):
    from lib.model_zoo.panorama import Windows, layout
    from vdb200 import ops
    lay = layout(Windows(size, stride, circular), H, W)
    ws = _tables(lay)
    x = np.random.default_rng(H * W + bs).standard_normal((bs, H, W, C)).astype(F32)
    dx = _dev(x)
    wins = [(int(oy), int(ox)) for oy in lay.oy for ox in lay.ox]
    for first, k in lay.chunks(3) + [(0, lay.nwin)]:
        ub = 1 if first % 2 == 0 else 0          # with a u block (CFG), the c block is a second copy
        out = torch.full(((ub + 1) * k * bs, lay.h, lay.w, C), float("nan"), device=DEV)
        ops.region_gather(dx, ws.oy, ws.ox, lay.h, lay.w, first, k, 0, ub, out=out)
        want = np.concatenate([_crop_nhwc(x, *wins[g], lay.h, lay.w) for g in range(first, first + k)])
        got = out.cpu().numpy()
        assert np.array_equal(got[:k * bs], want), (first, k)
        if ub:
            assert np.array_equal(got[k * bs:], want)


def merge_restated(eps, lay, wins, bs, halves, C):
    """The window average (vdb_region_merge_f32 at R = 0) in numpy fp32: ascending window index, first sets, later ones add
    (rounded), one division by the count"""
    H, W, h, w = lay.H, lay.W, lay.h, lay.w
    n = len(wins)
    e = eps.reshape(halves, n, bs, h, w, C)
    acc = np.zeros((halves, bs, H, W, C), dtype=F32)
    seen = np.zeros((H, W), dtype=bool)
    cnt = np.zeros((H, W), dtype=np.int64)
    for g, (oy, ox) in enumerate(wins):
        cols = (ox + np.arange(w)) % W
        rows = np.arange(oy, oy + h)
        blk = acc[:, :, oy:oy + h][:, :, :, cols]
        s = seen[np.ix_(rows, cols)][None, None, :, :, None]
        acc[:, :, oy:oy + h, cols] = np.where(s, blk + e[:, g], e[:, g])
        seen[np.ix_(rows, cols)] = True
        cnt[np.ix_(rows, cols)] += 1
    return (acc / cnt[None, None, :, :, None].astype(F32)).reshape(halves * bs, H, W, C), cnt


def merge_fp64(eps, lay, wins, bs, halves, C):
    n = len(wins)
    e = eps.astype(np.float64).reshape(halves, n, bs, lay.h, lay.w, C).transpose(1, 0, 2, 5, 3, 4)
    return P.average(list(e), wins, lay.h, lay.w, (halves, bs, C, lay.H, lay.W)).transpose(0, 1, 3, 4, 2).reshape(
        halves * bs, lay.H, lay.W, C)


@pytest.mark.parametrize("H,W,size,stride,circular", LAYOUTS)
@pytest.mark.parametrize("bs,halves,C", [(1, 2, 4), (2, 1, 4), (3, 2, 4), (2, 2, 5)])
def test_merge_with_no_regions_bitwise_and_against_fp64(H, W, size, stride, circular, bs, halves, C):
    from lib.model_zoo.panorama import Windows, layout
    from vdb200 import ops
    lay = layout(Windows(size, stride, circular), H, W)
    ws = _tables(lay)
    wins = [(int(oy), int(ox)) for oy in lay.oy for ox in lay.ox]
    n = lay.nwin
    eps = np.random.default_rng(n * 31 + bs).standard_normal((halves * n * bs, lay.h, lay.w, C)).astype(F32)
    want, cnt = merge_restated(eps, lay, wins, bs, halves, C)
    assert np.array_equal(cnt, lay.counts())
    ref = merge_fp64(eps, lay, wins, bs, halves, C)
    # eps of a chunk is [half 0 of its windows; half 1 of its windows]
    per_window = eps.reshape(halves, n, bs, lay.h, lay.w, C)
    outs = []
    for per in (n, 3, 1):
        out = torch.full((halves * bs, H, W, C), float("nan"), device=DEV)
        for first, k in lay.chunks(per):
            e = np.ascontiguousarray(per_window[:, first:first + k]).reshape(halves * k * bs, lay.h, lay.w, C)
            ops.region_merge(_dev(e), ws.oy, ws.ox, ws.cover_y, ws.cover_x, first, k, 0, None, out, halves=halves)
        outs.append(out.cpu().numpy())
    got = outs[0]
    assert np.array_equal(got, want), np.abs(got - want).max()
    for o in outs[1:]:
        assert np.array_equal(o, got), "chunked merges compute what one merge does"
    rel = np.abs(got - ref).max() / np.abs(ref).max()
    assert rel <= 1e-6, rel
    # single covering window: that window's eps bit for bit
    one = np.broadcast_to((cnt == 1)[None, :, :, None], got.shape)
    if one.any():
        assert np.array_equal(got[one], want[one])
    print(f"[panorama] merge {H}x{W} size {size} stride {stride} circular {circular} bs {bs} halves {halves}: "
          f"{n} windows, max count {cnt.max()}, rel err vs fp64 {rel:.2e}")


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


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


def _noise_fn(S, bs, C, H, W):
    """the inpainting blend's draws of grid index i, read back with the key the sampler drew -> NCHW"""
    from vdb200 import ops
    seed = S._st["seed"].clone()
    return lambda i: ops.inpaint_noise(seed, _idx(i), bs * H * W * C).view(bs, H, W, C).permute(0, 3, 1, 2).cpu()


@pytest.mark.parametrize("kind,H,W,stride,circular,multi,masked,per", [
    ("ddim", 16, 40, 8, False, False, False, 8), ("ddim", 32, 32, 8, False, True, False, 4), ("ddim", 16, 40, 8, True, False, False, 3),
    ("ddim", 16, 40, 8, False, False, True, 8), ("dpmpp", 16, 40, 8, False, False, False, 3), ("dpmpp", 32, 32, 8, True, True, False, 8),
    ("dpmpp", 16, 40, 8, False, False, True, 8)])
def test_sampler_vs_oracle(mini, monkeypatch, kind, H, W, stride, circular, multi, masked, per):
    from lib.model_zoo import panorama
    net, sd, gi = mini
    monkeypatch.setattr(panorama, "WINDOWS_PER_CHUNK", per)
    g = torch.Generator().manual_seed(H * W + stride + circular)
    bs, C, steps = 1, 4, 5
    xT = torch.randn(bs, C, H, W, generator=g)
    if multi:
        ct, ut = torch.randn(bs, 77, 768, generator=g) * 0.5, torch.randn(bs, 77, 768, generator=g) * 0.5
        ci, ui = torch.randn(bs, 257, 768, generator=g) * 0.5, torch.zeros(bs, 257, 768)
        conds, unconds, oracle_kw = [ct, ci], [ut, ui], dict(c_types=("text", "image"), ratios=[0.7, 0.3])
        cl = [_cinfo(ct, ut, ratio=0.7), _cinfo(ci, ui, typ="image", ratio=0.3)]
    else:
        conds, unconds, oracle_kw = [gi["c"][:bs]], [gi["u"][:bs]], {}
        cl = [_cinfo(conds[0], unconds[0])]
    x_info = {"type": "image", "xt": xT.to(DEV), "windows": panorama.Windows(16, stride, circular)}
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
    nwin = len(P.windows(H, W, 16, stride, circular)[2])
    ref = P.sample(sd, xT, conds, unconds, steps, 16, stride, circular, sampler=kind, order=2, scale=7.5, x0=x0, mask=mask,
                   noise_fn=_noise_fn(S, bs, C, H, W) if masked else None, model_channels=64, **oracle_kw)
    _cmp(x, ref, cos_min=0.999, tol=0.1, what=f"windowed {kind} {H}x{W} stride {stride} circular {circular} "
                                                f"{'dual' if multi else 'single'} {'masked ' if masked else ''}({nwin} windows, "
                                                f"chunks of {per}) vs oracle")
    if masked:
        keep = (mask == 0).expand(bs, C, H, W)
        assert torch.equal(x.cpu()[keep], x0.expand(bs, C, H, W)[keep]), "the kept region is x0 exactly"


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_invariants(mini, monkeypatch, kind):
    from lib.model_zoo import panorama
    net, sd, gi = mini
    g = torch.Generator().manual_seed(41)
    bs, C, H, W = 2, 4, 16, 40
    xT = torch.randn(bs, C, H, W, generator=g).to(DEV)
    c, u = gi["c"].repeat(bs, 1, 1).to(DEV), gi["u"].repeat(bs, 1, 1).to(DEV)

    def run(S, windows=None, cond=c, shape=(bs, C, H, W), xt=xT):
        x_info = {"type": "image", "xt": xt.clone()}
        if windows is not None:
            x_info["windows"] = windows
        with torch.no_grad():
            return S.sample(steps=6, shape=list(shape), x_info=x_info, c_info=_cinfo(cond, u, scale=5.0), verbose=False,
                            eta=0.)[0]

    # a window equal to the canvas: the unwindowed result, bit for bit, on the graph and the eager path
    Hs, Ws = 16, 24
    S0 = _sampler(kind, net)
    plain = run(S0, shape=(bs, C, Hs, Ws), xt=xT[..., :Ws].contiguous())
    S1 = _sampler(kind, net)
    one = run(S1, panorama.Windows(64, 8), shape=(bs, C, Hs, Ws), xt=xT[..., :Ws].contiguous())
    assert torch.equal(one, plain), "one window equal to the canvas gives the unwindowed result"
    assert torch.equal(run(_sampler(kind, net, use_cuda_graph=False), panorama.Windows(64, 8), shape=(bs, C, Hs, Ws),
                           xt=xT[..., :Ws].contiguous()), plain)
    print(f"[panorama] {kind} launches per step: unwindowed {S0.last_step_launches}, one window {S1.last_step_launches}")
    assert S1.last_step_launches == S0.last_step_launches + 2, "one gather and one merge"
    # graph against eager, a cached graph replayed on a new prompt against a fresh sampler, then other chunk sizes (their
    # samplers' context buffers evict this one's K / V^T projections from the per-layer cache)
    win = panorama.Windows(16, 8)
    Sg = _sampler(kind, net)
    g1 = run(Sg, win)
    assert torch.equal(g1, run(_sampler(kind, net, use_cuda_graph=False), win)), "graph path equals eager path"
    graph = next(iter(Sg._graphs.values()))[0]
    c2 = (torch.randn(bs, 77, 768, generator=g) * 0.5).to(DEV)
    g2 = run(Sg, win, cond=c2)
    assert next(iter(Sg._graphs.values()))[0] is graph, "the second call replays the cached graph"
    assert torch.equal(g2, run(_sampler(kind, net), win, cond=c2)), "replay on refilled contexts equals a fresh sampler"
    assert not torch.equal(g2, g1)
    assert torch.isfinite(g1).all()
    # the merge is the same for any chunking; the UNet's reductions are split by batch size, so other chunks change the last bits
    # of each window's eps, which a walk on the random-weight mini UNet amplifies (the oracle walks' tolerance)
    for per in (1, 3):
        monkeypatch.setattr(panorama, "WINDOWS_PER_CHUNK", per)
        _cmp(run(_sampler(kind, net), win), g1, cos_min=0.999, tol=0.1, what=f"{kind} chunks of {per} windows vs 8")
    monkeypatch.undo()


def test_wide_latent_through_the_vae_and_the_helper():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.panorama import Windows, panorama
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=True)
    z = torch.randn(1, 4, 8, 40, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        img = net.vae_decode(z.to(DEV), "image")
    assert img.shape == (1, 3, 64, 320)
    _cmp(img, O.vae_decode(sd, z), what="vae_decode of a 8x40 latent")
    gi = golden_inputs("mini")
    torch.manual_seed(0)
    out = panorama(net, DDIMSampler(net), _cinfo(gi["c"], gi["u"]), height=128, width=512, steps=5, windows=Windows(16, 8))
    assert out.shape == (1, 3, 128, 512) and torch.isfinite(out).all()
