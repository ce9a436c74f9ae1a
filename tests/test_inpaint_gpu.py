"""Inpainting on the GPU (lib/model_zoo/inpaint.py): vdb_inpaint_blend_f32 per element against its fp32 op-order restatement and
fp64, vdb_mask_to_latent against max-pooling, vdb_composite_f32, the Philox stream, the masked DDIM and DPM-Solver++ samplers on
the mini UNet against the oracle (oracle/inpaint_oracle.py) with the noises read back from vdb_inpaint_noise_f32, and the
sampler invariants: mask 0 returns x0, mask 1 returns the unmasked result, graph equals eager, a cached graph replays."""
import numpy as np
import pytest
import torch

from oracle import inpaint_oracle as I
from oracle import vd_oracle as O
from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
AC = O.ddpm_schedule(1000)["alphas_cumprod"]
F32 = np.float32


def restate(x, x0, m, z, a, b):
    """the header's op order in numpy fp32 (every op rounded to nearest)"""
    a, b = F32(a), F32(b)
    k = a * x0 + b * z
    return np.where(m == 1, x, np.where(m == 0, k, m * x + (F32(1) - m) * k))


def _soft_mask(g, shape):
    """uniform values with exact 0s and 1s mixed in"""
    m = g.random(shape).astype(F32)
    r = g.random(shape)
    m[r < 0.25] = 0.0
    m[r > 0.75] = 1.0
    return m


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("bs,per_item,dup,hw,c", [(1, False, False, 64 * 64, 4), (1, False, True, 35, 3), (4, True, True, 16 * 16, 4),
                                                  (4, False, True, 16 * 16, 4), (4, True, False, 9, 5)])
def test_blend_kernel_per_element(bs, per_item, dup, hw, c):
    from vdb200 import ops
    g = np.random.default_rng(bs * 1000 + hw)
    table = I.blend_rows(AC, O.make_ddim_timesteps(50)).astype(F32)
    d_table = _dev(table)
    worst = 0.0
    for idx in (49, 31, 1, 0):
        x = g.standard_normal((bs, hw, c)).astype(F32)
        x0 = (0.8 * g.standard_normal((bs, hw, c))).astype(F32)
        z = g.standard_normal((bs, hw, c)).astype(F32)
        m = _soft_mask(g, (bs if per_item else 1, hw))
        d_x = _dev(x)
        d_dup = torch.full_like(d_x, float("nan")) if dup else None
        ops.inpaint_blend(d_x, _dev(x0), _dev(m), d_table, _idx(idx), noise=_dev(z), x_dup=d_dup)
        mb = m[:, :, None]
        want = restate(x, x0, mb, z, *table[idx])
        got = d_x.cpu().numpy()
        assert np.array_equal(got, want), (idx, np.abs(got - want).max())
        if dup:
            assert np.array_equal(d_dup.cpu().numpy(), want)
        a, b = table[idx].astype(np.float64)
        ref = mb * x + (1 - mb.astype(np.float64)) * (a * x0 + b * z.astype(np.float64))
        rel = np.abs(got - ref).max() / np.abs(ref).max()
        worst = max(worst, rel)
        assert rel <= 1e-6, (idx, rel)
        if idx == 0:
            # the last row {1, 0}: the kept elements are x0 bit for bit, the generated ones the step's x bit for bit
            keep = np.broadcast_to(mb == 0, got.shape)
            gen = np.broadcast_to(mb == 1, got.shape)
            assert np.array_equal(got[keep], x0[keep]) and np.array_equal(got[gen], x[gen])
    print(f"[inpaint] blend bs {bs} per_item {per_item} hw {hw} c {c}: worst {worst:.3g} of max|x'| vs fp64")


def test_blend_with_philox_draws_recovers_the_noise_stream():
    """row {0, 1} and m = 0 turn the blend into z: the Philox draws of the blend equal vdb_inpaint_noise_f32 bit for bit, at the
    step index read from the device"""
    from vdb200 import ops
    bs, hw, c = 2, 33, 4
    n = bs * hw * c
    table = _dev(np.array([[0.0, 1.0]] * 8, dtype=F32))
    x0 = torch.randn(bs, hw, c, device=DEV)
    for step in (0, 5, 7):
        x = torch.randn(bs, hw, c, device=DEV)
        ops.inpaint_blend(x, x0, torch.zeros(hw, device=DEV), table, _idx(step), seed=_seed(987654321))
        z = ops.inpaint_noise(_seed(987654321), _idx(step), n)
        assert torch.equal(x.flatten(), z), step


def test_mask_to_latent_is_max_pool_and_composite_per_element():
    from lib.model_zoo.inpaint import composite, latent_mask
    g = np.random.default_rng(5)
    for n, H, W in ((1, 64, 64), (3, 5, 9)):
        m = _soft_mask(g, (n, 1, 8 * H, 8 * W))
        m[..., ::13, ::7] = 0.0
        got = latent_mask(_dev(m)).cpu()
        want = torch.nn.functional.max_pool2d(torch.from_numpy(m), 8)
        assert got.shape == (n, 1, H, W) and torch.equal(got, want)
    for n, mb in ((2, 2), (2, 1), (1, 1)):
        dec = g.uniform(-1, 1, (n, 3, 40, 24)).astype(F32)
        img = g.uniform(-1, 1, (n, 3, 40, 24)).astype(F32)
        m = _soft_mask(g, (mb, 1, 40, 24))
        got = composite(_dev(dec), _dev(img), _dev(m)).cpu().numpy()
        assert np.array_equal(got, np.where(m == 1, dec, np.where(m == 0, img, m * dec + (F32(1) - m) * img)))
        ref = m.astype(np.float64) * dec + (1 - m.astype(np.float64)) * img
        assert np.abs(got - ref).max() <= 1e-6
        keep = np.broadcast_to(m == 0, got.shape)
        assert np.array_equal(got[keep], img[keep])


def test_philox_stream():
    from scipy.stats import kstest
    from vdb200 import ops
    n = 1 << 20
    a = ops.inpaint_noise(_seed(1234), _idx(3), n)
    assert torch.equal(a, ops.inpaint_noise(_seed(1234), _idx(3), n)), "same seed and step must repeat bitwise"
    assert not torch.equal(a, ops.inpaint_noise(_seed(1235), _idx(3), n)), "different seeds must differ"
    b = ops.inpaint_noise(_seed(1234), _idx(4), n)
    assert not torch.equal(a, b), "different steps must differ"
    assert torch.equal(a[:1001], ops.inpaint_noise(_seed(1234), _idx(3), 1001)), "a prefix is the same stream"
    z = a.double().cpu().numpy()
    mean, var = z.mean(), z.var()
    stat, p = kstest(z, "norm")
    adj_e = np.corrcoef(z[:-1], z[1:])[0, 1]
    adj_pair = np.corrcoef(z[0::2], z[1::2])[0, 1]          # the two members of one Box-Muller pair
    adj_s = np.corrcoef(z, b.double().cpu().numpy())[0, 1]
    print(f"[inpaint] Philox over {n} draws: mean {mean:.2e} var {var:.5f} KS {stat:.2e} (p {p:.3f}) "
          f"corr(elem, elem+1) {adj_e:.1e} corr(pair) {adj_pair:.1e} corr(step, step+1) {adj_s:.1e}")
    se = 1.0 / np.sqrt(n)
    assert abs(mean) <= 5 * se and abs(var - 1) <= 5 * np.sqrt(2.0) * se
    assert p > 1e-3
    for r in (adj_e, adj_pair, adj_s):
        assert abs(r) <= 5 * se
    assert np.isfinite(z).all() and np.abs(z).max() < 7


# ---- the samplers on the mini UNet -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale=7.5, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _sampler(kind, net):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return DDIMSampler(net) if kind == "ddim" else DPMSolverSampler(net, order=2)


def _noise_fn(S, bs, C, H, W):
    """the sampler's draws of grid index i, read back through vdb_inpaint_noise_f32 with the key it drew -> NCHW"""
    from vdb200 import ops
    seed = S._st["seed"].clone()
    return lambda i: ops.inpaint_noise(seed, _idx(i), bs * H * W * C).view(bs, H, W, C).permute(0, 3, 1, 2).cpu()


def _masks(bs, H, W):
    """a soft latent mask per item: keep the left part, regenerate the right, a soft band between"""
    m = torch.zeros(bs, 1, H, W)
    for b in range(bs):
        m[b, :, :, W // 2 + b:] = 1.0
        m[b, :, :, W // 2 - 2 + b] = 0.3
        m[b, :, :, W // 2 - 1 + b] = 0.7
    return m


@pytest.mark.parametrize("kind,start,multi", [("ddim", "full", False), ("ddim", "k", False), ("ddim", "full", True),
                                              ("dpmpp", "full", False), ("dpmpp", "k", False), ("dpmpp", "full", True)])
def test_sampler_vs_oracle(mini, kind, start, multi):
    net, sd, gi = mini
    g = torch.Generator().manual_seed(17)
    bs, C, H, W = 2, 4, 16, 16
    # a batch-1 x0 is broadcast over the batch (the img2img start noises it once per item with the injected draws)
    x0 = torch.randn(bs if (kind, start) == ("ddim", "k") else 1, C, H, W, generator=g) * 0.8
    xT = torch.randn(bs, C, H, W, generator=g)
    q_noise = torch.randn(bs, C, H, W, generator=g)
    steps, k = 8, 5
    if multi:
        ct, ut = torch.randn(bs, 77, 768, generator=g) * 0.5, torch.randn(bs, 77, 768, generator=g) * 0.5
        ci, ui = torch.randn(bs, 257, 768, generator=g) * 0.5, torch.zeros(bs, 257, 768)
        conds, unconds, oracle_kw = [ct, ci], [ut, ui], dict(c_types=("text", "image"), ratios=[0.7, 0.3])
        cl = [_cinfo(ct, ut, ratio=0.7), _cinfo(ci, ui, typ="image", ratio=0.3)]
    else:
        conds, unconds, oracle_kw = [gi["c"].repeat(bs, 1, 1)], [gi["u"].repeat(bs, 1, 1)], {}
        cl = [_cinfo(conds[0], unconds[0])]
    # the first case converts a pixel mask on the device; the others pass the latent mask
    lat = _masks(bs, H, W)
    mask = lat.repeat_interleave(8, 2).repeat_interleave(8, 3) if (kind, start, multi) == ("ddim", "full", False) else lat
    x_info = {"type": "image", "x0": x0.to(DEV), "inpaint_mask": mask.to(DEV)}
    if start == "k":
        x_info["x0_forward_timesteps"] = k
    else:
        x_info["xt"] = xT.to(DEV)
    S = _sampler(kind, net)
    orig = net.q_sample
    net.q_sample = lambda x_start, t, noise_=None: orig(x_start, t, noise=q_noise.to(x_start.device))   # inject the draw
    try:
        with torch.no_grad():
            kw = dict(steps=steps, shape=[bs, C, H, W], x_info=x_info, verbose=False, eta=0.)
            x, inter = S.sample_multicontext(c_info_list=cl, **kw) if multi else S.sample(c_info=cl[0], **kw)
    finally:
        net.q_sample = orig
    ref = I.sample(sd, xT, conds, unconds, steps, x0, lat, _noise_fn(S, bs, C, H, W), sampler=kind, order=2, scale=7.5,
                   x0_forward_timesteps=k if start == "k" else None, x0_noise=q_noise, model_channels=64, **oracle_kw)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"masked {kind} ({start} start, {'dual' if multi else 'single'} context) vs oracle")
    keep = (lat == 0).expand(bs, C, H, W)
    assert torch.equal(x.cpu()[keep], x0.expand(bs, C, H, W)[keep]), "the kept region is x0 exactly"


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_invariants(mini, kind):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    net, sd, gi = mini
    cls = DDIMSampler if kind == "ddim" else DPMSolverSampler
    g = torch.Generator().manual_seed(23)
    bs, C, H, W = 2, 4, 16, 16
    x0 = (torch.randn(bs, C, H, W, generator=g) * 0.8).to(DEV)
    xT = torch.randn(bs, C, H, W, generator=g).to(DEV)
    c, u = gi["c"].repeat(bs, 1, 1).to(DEV), gi["u"].repeat(bs, 1, 1).to(DEV)

    def run(S, mask=None, x0_=x0, seed=0, k=None):
        x_info = {"type": "image"}
        if mask is not None:
            x_info.update(x0=x0_, inpaint_mask=mask.to(DEV))
        if k is None:
            x_info["xt"] = xT.clone()
        else:                                   # the img2img start (an injected x_T would take precedence over it)
            x_info["x0_forward_timesteps"] = k
        torch.manual_seed(seed)
        with torch.no_grad():
            return S.sample(steps=6, shape=[bs, C, H, W], x_info=x_info, c_info=_cinfo(c, u, scale=5.0), verbose=False, eta=0.)[0]

    S0 = cls(net)
    plain = run(S0)
    Sm = cls(net)
    assert torch.equal(run(Sm, torch.zeros(1, 1, H, W)), x0), "mask 0: the result is x0 bit for bit"
    assert torch.equal(run(Sm, torch.zeros(bs, 1, H, W), k=4), x0), "mask 0 from the img2img start too"
    assert torch.equal(run(Sm, torch.ones(bs, 1, H, W)), plain), "mask 1: the unmasked result bit for bit"
    print(f"[inpaint] {kind} launches per step: unmasked {S0.last_step_launches}, masked {Sm.last_step_launches}")
    assert Sm.last_step_launches == S0.last_step_launches + 1
    # graph against eager, and a second call with a new image, mask and seed on the cached graph against a fresh sampler
    mask = _masks(bs, H, W)
    Sg = cls(net)
    eager = run(cls(net, use_cuda_graph=False), mask, seed=1)
    g1 = run(Sg, mask, seed=1)
    assert torch.equal(eager, g1), "graph path must be bit-identical to the eager path"
    graph = next(iter(Sg._graphs.values()))[0]
    x0b = (torch.randn(bs, C, H, W, generator=g) * 0.8).to(DEV)
    mask2 = torch.flip(mask, dims=[3])
    g2 = run(Sg, mask2, x0_=x0b, seed=2)
    assert next(iter(Sg._graphs.values()))[0] is graph, "the second call replays the cached graph"
    assert torch.equal(g2, run(cls(net), mask2, x0_=x0b, seed=2)), "replay on refilled buffers must equal a fresh sampler"
    assert torch.equal(g2, run(cls(net, use_cuda_graph=False), mask2, x0_=x0b, seed=2))
    assert not torch.equal(g2, run(cls(net), mask2, x0_=x0b, seed=3)), "the seed reaches the draws"
    # a broadcast mask is another graph (mask_per_item is in the key) with the per-item result of the same mask
    g3 = run(Sg, mask[:1], seed=4)
    assert torch.equal(g3, run(cls(net), mask[:1].expand(bs, 1, H, W).contiguous(), seed=4))


def test_inpaint_wrapper_with_the_vae():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.inpaint import inpaint
    from oracle.make_golden import golden_inputs
    net, _ = build_net(mini=True, with_vae=True)
    gi = golden_inputs("mini")
    g = torch.Generator().manual_seed(29)
    image = torch.rand(1, 3, 128, 128, generator=g).to(DEV)        # [0, 1], as ToTensor gives it
    mask = torch.zeros(1, 1, 128, 128)
    mask[..., 40:90, 50:100] = 1.0
    mask = mask.to(DEV)
    torch.manual_seed(0)
    out = inpaint(net, DDIMSampler(net), image, mask, _cinfo(gi["c"], gi["u"]), steps=5)
    assert out.shape == image.shape and torch.isfinite(out).all()
    keep = (mask == 0).expand_as(image)
    assert torch.equal(out[keep], image[keep]), "paste-back keeps the original pixels outside the mask"
    torch.manual_seed(0)
    raw = inpaint(net, DDIMSampler(net), image, mask, _cinfo(gi["c"], gi["u"]), steps=5, paste_back=False)
    gen = (mask == 1).expand_as(image)
    assert torch.equal(out[gen], raw[gen])
