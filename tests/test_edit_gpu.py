"""Editing on the GPU (lib/model_zoo/edit.py): vdb_ddim_cfg_step with an inversion row undone by the forward row,
vdb_latent_store_slot_f32, vdb_inversion_blend_f32 against its fp32 op-order restatement and fp64, vdb_diffedit_mask_f32 against
the fp64 rule; on the mini UNet the inversion walk and the trajectory-blended DDIM / DPM-Solver++ walks against
oracle/edit_oracle.py; and the invariants: mask 0 returns x0, mask 1 the unmasked walk, graph equals eager, edit with src == tgt
keeps x0, and a second edit call replays the cached graphs."""
import numpy as np
import pytest
import torch

from oracle import edit_oracle as E
from oracle import vd_oracle as O
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


def _soft_mask(g, shape):
    m = g.random(shape).astype(F32)
    r = g.random(shape)
    m[r < 0.25] = 0.0
    m[r > 0.75] = 1.0
    return m


def test_inversion_row_then_forward_row_is_the_identity():
    from lib.model_zoo.edit import inversion_rows
    from vdb200 import ops
    sched = O.ddim_schedule(O.ddpm_schedule(1000)["alphas_cumprod"], 50)
    inv = _dev(inversion_rows(sched["alphas"], sched["alphas_prev"], 50))
    fwd = _dev(np.stack([sched["alphas"], sched["alphas_prev"], np.zeros(50, F32), sched["sqrt_one_minus_alphas"]], 1).astype(F32))
    g = torch.Generator().manual_seed(3)
    n = 4 * 32 * 32 * 4
    x = torch.randn(n, generator=g).to(DEV)
    e = torch.randn(n, generator=g).to(DEV)
    worst = 0.0
    for i in (0, 1, 24, 49):
        y, _ = ops.ddim_cfg_step(None, e, x, inv, 1.0, step_idx=_idx(i))
        back, _ = ops.ddim_cfg_step(None, e, y, fwd, 1.0, step_idx=_idx(i))
        rel = ((back - x).abs().max() / x.abs().max()).item()
        worst = max(worst, rel)
        assert rel <= 4e-6, (i, rel)
    print(f"[edit] inversion row then forward row: worst {worst:.3g} of max|x|")


def test_store_slot_writes_exactly_one_slot():
    from vdb200 import ops
    for shape in ((2, 8, 8, 4), (3, 5, 7)):          # n % 4 == 0 and an odd n
        slots = 5
        x = torch.randn(*shape, device=DEV)
        for idx, off in ((0, 1), (2, 1), (3, 0), (4, 1), (-1, 0)):
            ring = torch.full((slots,) + shape, float("nan"), device=DEV)
            ops.latent_store_slot(x, ring, _idx(idx), off)
            s = idx + off
            for j in range(slots):
                if j == s:
                    assert torch.equal(ring[j], x), (shape, idx, off)
                else:
                    assert torch.isnan(ring[j]).all(), (shape, idx, off, j)


@pytest.mark.parametrize("bs,per_item,dup,hw,c", [(1, False, False, 64 * 64, 4), (2, True, True, 16 * 16, 4),
                                                  (4, False, True, 16 * 16, 4), (3, True, False, 9, 5)])
def test_inversion_blend_per_element(bs, per_item, dup, hw, c):
    from vdb200 import ops
    g = np.random.default_rng(bs * 100 + hw)
    slots = 6
    ring = g.standard_normal((slots, bs, hw, c)).astype(F32)
    d_ring = _dev(ring)
    for idx in (5, 2, 0):
        x = g.standard_normal((bs, hw, c)).astype(F32)
        m = _soft_mask(g, (bs if per_item else 1, hw))
        d_x = _dev(x)
        d_dup = torch.full_like(d_x, float("nan")) if dup else None
        ops.inversion_blend(d_x, d_ring, _dev(m), _idx(idx), x_dup=d_dup)
        mb = m[:, :, None]
        k = ring[idx]
        want = np.where(mb == 1, x, np.where(mb == 0, k, mb * x + (F32(1) - mb) * k))
        got = d_x.cpu().numpy()
        assert np.array_equal(got, want), (idx, np.abs(got - want).max())
        if dup:
            assert np.array_equal(d_dup.cpu().numpy(), want)
        ref = mb * x.astype(np.float64) + (1 - mb.astype(np.float64)) * k
        assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()
        keep, gen = np.broadcast_to(mb == 0, got.shape), np.broadcast_to(mb == 1, got.shape)
        assert np.array_equal(got[keep], k[keep]) and np.array_equal(got[gen], x[gen])
    # a counter outside [0, slots) reads no slot and leaves x and x_dup as they are
    x = g.standard_normal((bs, hw, c)).astype(F32)
    m = _dev(np.zeros((bs if per_item else 1, hw), F32))
    for idx in (slots, -1):
        d_x = _dev(x)
        d_dup = torch.full_like(d_x, float("nan")) if dup else None
        ops.inversion_blend(d_x, d_ring, m, _idx(idx), x_dup=d_dup)
        assert np.array_equal(d_x.cpu().numpy(), x), idx
        if dup:
            assert torch.isnan(d_dup).all(), idx


def _mix(u, c, s):
    return c if u is None else u + F32(s) * (c - u)


@pytest.mark.parametrize("D,bs,H,W,cfg_src,cfg_tgt", [(10, 2, 16, 16, False, True), (3, 1, 64, 64, True, True),
                                                      (1, 3, 5, 7, False, False)])
def test_diffedit_mask_kernel(D, bs, H, W, cfg_src, cfg_tgt):
    from vdb200 import ops
    g = np.random.default_rng(D * 10 + bs)
    C = 4
    shp = (D * bs, H, W, C)
    su = g.standard_normal(shp).astype(F32) if cfg_src else None
    sc = g.standard_normal(shp).astype(F32)
    tu = g.standard_normal(shp).astype(F32) if cfg_tgt else None
    tc = g.standard_normal(shp).astype(F32)
    # a planted region of large disagreement per image
    for b in range(bs):
        tc.reshape(D, bs, H, W, C)[:, b, b:b + H // 2, :W // 2] += 4.0
    s_src, s_tgt = (5.0 if cfg_src else 1.0), (7.5 if cfg_tgt else 1.0)
    t = lambda a: None if a is None else _dev(a)
    got = ops.diffedit_mask(t(su), t(sc), s_src, t(tu), t(tc), s_tgt, D, 3.0).cpu().numpy()
    assert got.shape == (bs, H, W)
    again = ops.diffedit_mask(t(su), t(sc), s_src, t(tu), t(tc), s_tgt, D, 3.0).cpu().numpy()
    assert np.array_equal(got, again), "bit-reproducible"
    es = _mix(su, sc, s_src).astype(np.float64).reshape(D, bs, H, W, C).transpose(0, 1, 4, 2, 3)
    et = _mix(tu, tc, s_tgt).astype(np.float64).reshape(D, bs, H, W, C).transpose(0, 1, 4, 2, 3)
    want, d, cap = E.diffedit_mask(es, et)
    near = np.abs(np.minimum(d[:, 0], cap[:, None, None]) / cap[:, None, None] - 0.5) < 1e-5
    agree = (got == want[:, 0]) | near
    assert agree.all(), int((~agree).sum())
    assert set(np.unique(got)) <= {0.0, 1.0} and got.any()
    # identical sides: cap == 0, all 0
    zero = ops.diffedit_mask(t(su), t(sc), s_src, t(su), t(sc), s_src, D, 3.0).cpu().numpy()
    assert not zero.any()
    # the front end's own refusals: no draws, and an out of the wrong size
    with pytest.raises(ValueError, match="D must be >= 1"):
        ops.diffedit_mask(t(su), t(sc), s_src, t(tu), t(tc), s_tgt, 0, 3.0)
    for n_out in (bs * H * W - 1, bs * H * W + 1):
        with pytest.raises(ValueError, match="out: expected"):
            ops.diffedit_mask(t(su), t(sc), s_src, t(tu), t(tc), s_tgt, D, 3.0, out=torch.empty(n_out, device=DEV))


# ---- the walks on the mini UNet -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=7.5, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _contexts(gi, bs, multi, g):
    if multi:
        ct, ut = torch.randn(bs, 77, 768, generator=g) * 0.5, torch.randn(bs, 77, 768, generator=g) * 0.5
        ci, ui = torch.randn(bs, 257, 768, generator=g) * 0.5, torch.zeros(bs, 257, 768)
        return [ct, ci], [ut, ui], dict(c_types=("text", "image"), ratios=[0.7, 0.3]), \
            lambda s: [_cinfo(ct, ut, s, ratio=0.7), _cinfo(ci, ui, s, typ="image", ratio=0.3)]
    c, u = gi["c"].repeat(bs, 1, 1), gi["u"].repeat(bs, 1, 1)
    return [c], [u], {}, lambda s: [_cinfo(c, u, s)]


def _invert(S, steps, x0, cl, k):
    return S.invert_multicontext(steps, x0.to(DEV), cl, k=k) if len(cl) > 1 else S.invert(steps, x0.to(DEV), cl[0], k=k)


def _sample(S, steps, shape, x_info, cl):
    kw = dict(steps=steps, shape=shape, x_info=x_info, verbose=False, eta=0.)
    with torch.no_grad():
        return (S.sample_multicontext(c_info_list=cl, **kw) if len(cl) > 1 else S.sample(c_info=cl[0], **kw))[0]


@pytest.mark.parametrize("k,multi", [(None, False), (5, False), (None, True), (5, True)])
def test_inversion_vs_oracle(mini, k, multi):
    from lib.model_zoo.ddim import DDIMSampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(31)
    bs, C, H, W, steps = 2, 4, 16, 16, 8
    x0 = torch.randn(1, C, H, W, generator=g) * 0.8          # a batch-1 x0 is broadcast over the contexts' batch
    conds, unconds, okw, cl = _contexts(gi, bs, multi, g)
    S = DDIMSampler(net)
    inv = _invert(S, steps, x0, cl(1.0), k)
    kk = 8 if k is None else k
    assert inv.k == kk and inv.trajectory.shape == (kk + 1, bs, H, W, C)
    traj = inv.trajectory.permute(0, 1, 4, 2, 3).cpu()
    assert torch.equal(traj[0], x0.expand(bs, C, H, W)), "slot 0 is x0"
    assert torch.equal(inv.xt.cpu(), traj[kk])
    ref = E.invert(sd, x0.expand(bs, C, H, W), conds, unconds, steps, k=kk, scale=1.0, model_channels=64, **okw)
    for i in (1, kk // 2, kk):
        _cmp(traj[i], ref[i], cos_min=0.995, tol=0.1, what=f"inversion slot {i} of {kk} ({'dual' if multi else 'single'})")
    # graph against eager
    eager = _invert(DDIMSampler(net, use_cuda_graph=False), steps, x0, cl(1.0), k)
    assert torch.equal(eager.trajectory, inv.trajectory), "graph path must be bit-identical to the eager path"


@pytest.mark.parametrize("kind,multi", [("ddim", False), ("ddim", True), ("dpmpp", False)])
def test_sample_from_inversion_vs_oracle(mini, kind, multi):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    g = torch.Generator().manual_seed(37)
    bs, C, H, W, steps, k = 2, 4, 16, 16, 8, 6
    x0 = torch.randn(bs, C, H, W, generator=g) * 0.8
    conds, unconds, okw, cl = _contexts(gi, bs, multi, g)
    inv = _invert(DDIMSampler(net), steps, x0, cl(1.0), k)
    lat = torch.zeros(bs, 1, H, W)
    lat[0, :, :, W // 2:] = 1.0
    lat[1, :, H // 2:, :] = 1.0
    lat[:, :, 3, 3] = 0.4
    S = DDIMSampler(net) if kind == "ddim" else DPMSolverSampler(net, order=2)
    x = _sample(S, steps, [bs, C, H, W], {"type": "image", "inversion": inv, "inpaint_mask": lat.to(DEV)}, cl(3.0))
    traj = inv.trajectory.permute(0, 1, 4, 2, 3).cpu()
    ref = E.sample(sd, traj, conds, unconds, steps, mask=lat, sampler=kind, order=2, scale=3.0, model_channels=64, **okw)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"{kind} from an inversion, masked ({'dual' if multi else 'single'})")
    keep = (lat == 0).expand(bs, C, H, W)
    assert torch.equal(x.cpu()[keep], x0[keep]), "the kept region is x0 exactly"
    eager = _sample(type(S)(net, use_cuda_graph=False) if kind == "ddim" else DPMSolverSampler(net, order=2, use_cuda_graph=False),
                    steps, [bs, C, H, W], {"type": "image", "inversion": inv, "inpaint_mask": lat.to(DEV)}, cl(3.0))
    assert torch.equal(eager, x), "graph path must be bit-identical to the eager path"


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_invariants(mini, kind):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    make = (lambda **kw: DDIMSampler(net, **kw)) if kind == "ddim" else (lambda **kw: DPMSolverSampler(net, order=2, **kw))
    g = torch.Generator().manual_seed(41)
    bs, C, H, W, steps = 2, 4, 16, 16, 6
    x0 = (torch.randn(bs, C, H, W, generator=g) * 0.8).to(DEV)
    c, u = gi["c"].repeat(bs, 1, 1), gi["u"].repeat(bs, 1, 1)
    inv = DDIMSampler(net).invert(steps, x0, _cinfo(c, u, 1.0), k=4)
    shape = [bs, C, H, W]

    def run(S, mask=None, inv_=inv):
        x_info = {"type": "image", "inversion": inv_}
        if mask is not None:
            x_info["inpaint_mask"] = mask.to(DEV)
        return _sample(S, steps, shape, x_info, [_cinfo(c, u, 5.0)])

    S0, Sm = make(), make()
    plain = run(S0)
    assert torch.equal(run(Sm, torch.zeros(1, 1, H, W)), x0), "mask 0: the result is x0 bit for bit"
    assert torch.equal(run(Sm, torch.ones(bs, 1, H, W)), plain), "mask 1: the unmasked walk bit for bit"
    print(f"[edit] {kind} launches per step: unmasked {S0.last_step_launches}, masked {Sm.last_step_launches}")
    assert Sm.last_step_launches == S0.last_step_launches + 1
    # a cached graph replays on a new inversion and mask, and equals a fresh sampler
    mask = torch.zeros(bs, 1, H, W)
    mask[..., 4:12, 2:10] = 1.0
    Sg = make()
    g1 = run(Sg, mask)
    graph = next(iter(Sg._graphs.values()))[0]
    x0b = (torch.randn(bs, C, H, W, generator=g) * 0.8).to(DEV)
    inv2 = DDIMSampler(net).invert(steps, x0b, _cinfo(c, u, 1.0), k=4)
    g2 = run(Sg, torch.flip(mask, dims=[3]), inv2)
    assert next(iter(Sg._graphs.values()))[0] is graph, "the second call replays the cached graph"
    assert torch.equal(g2, run(make(), torch.flip(mask, dims=[3]), inv2))
    assert torch.equal(g2, run(make(use_cuda_graph=False), torch.flip(mask, dims=[3]), inv2))
    assert not torch.equal(g1, g2)


def test_edit_src_equals_tgt_and_graph_reuse():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.edit import edit
    from oracle.make_golden import golden_inputs
    net, _ = build_net(mini=True, with_vae=True)
    gi = golden_inputs("mini")
    g = torch.Generator().manual_seed(43)
    n = 2
    image = torch.rand(n, 3, 128, 128, generator=g).to(DEV)
    ci = _cinfo(gi["c"].repeat(n, 1, 1), gi["u"].repeat(n, 1, 1), 7.5)
    decoded, encoded = [], []
    orig, orig_enc = net.vae_decode, net.vae_encode
    net.vae_decode = lambda z, which, **kw: (decoded.append(z.clone()), orig(z, which, **kw))[1]
    net.vae_encode = lambda x, which, **kw: (lambda z: (encoded.append(z.clone()), z)[1])(orig_enc(x, which, **kw))
    try:
        S = DDIMSampler(net)
        torch.manual_seed(0)
        out, mask = edit(net, S, image, ci, ci, steps=10, strength=0.5, mask='auto', n_draws=4)
        assert out.shape == image.shape and torch.isfinite(out).all()
        assert mask.shape == (n, 1, 16, 16) and not mask.any(), "src == tgt: an all-zero mask"
        assert torch.equal(decoded[-1], encoded[-1]), "mask 0 everywhere: the latent is x0"
        # a second call of the same shapes replays the cached graphs and captures nothing
        g_inv, g_fwd = next(iter(S._inv_graphs.values()))[0], next(iter(S._graphs.values()))[0]
        image2 = torch.rand(n, 3, 128, 128, generator=g).to(DEV)
        tgt = _cinfo(gi["c"].repeat(n, 1, 1) * 0.5, gi["u"].repeat(n, 1, 1), 7.5)
        # the eager step that precedes every capture sets these; a call that only replays leaves them alone
        S.last_step_launches = S.last_invert_step_launches = None
        torch.manual_seed(1)
        out2, mask2 = edit(net, S, image2, ci, tgt, steps=10, strength=0.5, mask='auto', n_draws=4)
        assert next(iter(S._inv_graphs.values()))[0] is g_inv and next(iter(S._graphs.values()))[0] is g_fwd
        assert S.last_step_launches is None and S.last_invert_step_launches is None, "no eager step: nothing was captured"
        assert torch.isfinite(out2).all() and set(mask2.unique().tolist()) <= {0.0, 1.0}
        keep = (mask2 == 0).expand(n, 4, 16, 16)
        assert torch.equal(decoded[-1][keep], encoded[-1][keep]), "outside the mask the latent is x0"
    finally:
        net.vae_decode, net.vae_encode = orig, orig_enc
