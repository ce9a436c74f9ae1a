"""Self-attention guidance on the GPU (lib/model_zoo/sag.py): the key mass against fp64 from the same bf16 operands in both
self-attention layouts, the degrade against an fp64 restatement, the guide bitwise, and the DDIM / DPM-Solver++ SAG walks of the
mini UNet against oracle/sag_oracle.py, with CFG and without, one context and two, and with an inpainting mask; the graph path
against the eager path bit for bit, and a cached graph replayed on new prompts."""
import numpy as np
import pytest
import torch

from test_parity_gpu import _cmp, build_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32


def _idx(i):
    return torch.tensor([i], dtype=torch.int32, device=DEV)


# ---- vdb_sattn_key_mass_f32 ------------------------------------------------------------------------------------------------------
def _key_mass_fp64(q, k, B, H, N, d, dk, scale):
    """sum_h sum_p softmax_j(scale q . k) per item and key, fp64 from q [B, N, H, dk] and k [B, N, H, dk] (bf16 values)"""
    q, k = q[..., :d].double(), k[..., :d].double()
    p = torch.softmax(torch.einsum("bphc,bjhc->bhpj", q, k) * scale, dim=-1)
    return p.sum(dim=(1, 2))


@pytest.mark.parametrize("layout", ["fused", "padded"])
@pytest.mark.parametrize("N", [64, 30, 256, 1024])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_key_mass_against_fp64(d, N, layout):
    from vdb200 import ops
    g = torch.Generator(device=DEV).manual_seed(1000 * d + N)
    B, H, row0, n, w = 3, 8, 1, 2, 0.37
    dk = ops.attention_pads(d)[0]
    scale = d ** -0.5
    # random values in the head padding columns too: the kernel must read only the first d of each head's dk
    rnd = lambda *s: (torch.randn(*s, generator=g, device=DEV) * 1.5).to(torch.bfloat16)
    if layout == "fused":
        qk = rnd(B * N, 2 * H * dk)
        q, k, kw = qk, qk, dict(q_col0=0, k_col0=H * dk)
        qv, kv = qk[:, :H * dk].view(B, N, H, dk), qk[:, H * dk:].view(B, N, H, dk)
    else:
        Np = (N + 7) // 8 * 8
        q, k = rnd(B * N, H * dk), rnd(B * Np, H * dk)
        kw = dict(kv_bstride=Np)
        qv, kv = q.view(B, N, H, dk), k.view(B, Np, H, dk)[:, :N]
    mass0 = torch.rand(n, N, generator=g, device=DEV)
    got = ops.sattn_key_mass(q, k, mass0.clone(), row0, H, N, d, w=w, scale=scale, **kw)
    again = ops.sattn_key_mass(q, k, mass0.clone(), row0, H, N, d, w=w, scale=scale, **kw)
    assert torch.equal(got, again), "the key mass must be bit-reproducible"
    ref = mass0.double() + w * _key_mass_fp64(qv, kv, B, H, N, d, dk, scale)[row0:row0 + n]
    err = (got.double() - ref).abs().max().item()
    print(f"[sag] key mass d {d} N {N} {layout}: max|err| {err:.3g} of max {ref.abs().max().item():.3g}")
    assert err <= 1e-5 * max(1.0, ref.abs().max().item()) * H


# ---- vdb_sag_degrade_f32 and vdb_sag_guide_f32 --------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(64, 64), (40, 48)])
@pytest.mark.parametrize("kind", ["soft", "zero", "one"])
def test_degrade_against_fp64(H, W, kind):
    from lib.model_zoo.sag import mid_size
    from oracle import sag_oracle as S
    from vdb200 import ops
    g = torch.Generator().manual_seed(H * W + len(kind))
    bs, C = 3, 4
    hm, wm = mid_size(H, W)
    x = torch.randn(bs, H, W, C, generator=g)
    e = torch.randn(bs, H, W, C, generator=g)
    mass = {"soft": 0.5 + torch.rand(bs, hm * wm, generator=g), "zero": torch.zeros(bs, hm * wm),
            "one": torch.full((bs, hm * wm), 2.0)}[kind]
    a = np.array([0.9, 0.5, 0.3, 0.07])
    table = torch.from_numpy(np.stack([np.sqrt(a), np.sqrt(1 - a)], 1).astype(F32))
    got = ops.sag_degrade(x.to(DEV), e.to(DEV), mass.to(DEV), table.to(DEV), _idx(2), hm, wm).cpu()
    sa, s1 = table[2].tolist()
    if kind == "zero":          # no cell marked: the re-noise of x0, in the kernel's fp32 op order
        xn, en = x.numpy(), e.numpy()
        x0 = (xn - F32(s1) * en) / F32(sa)
        want = F32(sa) * x0 + F32(s1) * en
        assert np.array_equal(got.numpy(), want), "an all-zero mask gives the re-noise of x0 bit for bit"
    xd, ed = x.double().permute(0, 3, 1, 2), e.double().permute(0, 3, 1, 2)
    M = (mass > 1.0).double().view(bs, 1, hm, wm)[:, :, S.nearest_index(H, hm)][:, :, :, S.nearest_index(W, wm)]
    x0 = (xd - s1 * ed) / sa
    ref = (sa * (M * S.blur(x0) + (1 - M) * x0) + s1 * ed).permute(0, 2, 3, 1)
    err = (got.double() - ref).abs().max().item()
    print(f"[sag] degrade {H}x{W} {kind}: max|err| {err:.3g}")
    assert err <= 2e-6 * ref.abs().max().item()


@pytest.mark.parametrize("cfg", [True, False])
def test_guide_bitwise(cfg):
    from vdb200 import ops
    g = torch.Generator().manual_seed(5)
    n, s = 2 * 64 * 64 * 4 + 3, 0.75
    e_u, e_c, e_deg = (torch.randn(n, generator=g) for _ in range(3))
    gu, gc = e_u.to(DEV), e_c.to(DEV)
    ops.sag_guide(gu if cfg else None, gc, e_deg.to(DEV), s)
    src = (e_u if cfg else e_c).numpy()
    d = F32(s) * (src - e_deg.numpy())
    assert np.array_equal(gc.cpu().numpy(), e_c.numpy() + d)
    assert np.array_equal(gu.cpu().numpy(), e_u.numpy() + d if cfg else e_u.numpy())


# ---- the SAG walks on the mini UNet ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mini():
    from oracle.make_golden import golden_inputs
    net, sd = build_net(mini=True, with_vae=False)
    return net, sd, golden_inputs("mini")


def _cinfo(c, u, scale, typ="text", **kw):
    return dict({"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV),
                 "unconditional_guidance_scale": scale}, **kw)


def _sampler(kind, net, **kw):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return DDIMSampler(net, **kw) if kind == "ddim" else DPMSolverSampler(net, order=2, **kw)


def _contexts(gi, g, bs, multi):
    if multi:
        ct, ut = torch.randn(bs, 77, 768, generator=g) * 0.5, torch.randn(bs, 77, 768, generator=g) * 0.5
        ci, ui = torch.randn(bs, 257, 768, generator=g) * 0.5, torch.zeros(bs, 257, 768)
        return [ct, ci], [ut, ui], dict(c_types=("text", "image"), ratios=[0.7, 0.3]), [0.7, 0.3]
    return [gi["c"].repeat(bs, 1, 1)], [gi["u"].repeat(bs, 1, 1)], {}, [1.0]


def _cinfos(conds, unconds, scale, ratios):
    types = ["text", "image"]
    return [_cinfo(c, u, scale, typ=types[i], ratio=r) for i, (c, u, r) in enumerate(zip(conds, unconds, ratios))]


# (sampler, CFG scale, two contexts, latent side, steps, seed): the sides give mid maps of 4 x 4 (fused q | k) and 3 x 3 (padded
# keys); each seed keeps every oracle mass at least 1e-3 from the threshold
WALKS = [("ddim", 7.5, False, 32, 4, 18), ("dpmpp", 7.5, False, 24, 4, 17), ("ddim", 1.0, False, 32, 4, 17),
         ("dpmpp", 1.0, False, 24, 4, 19), ("ddim", 7.5, True, 24, 4, 17), ("dpmpp", 7.5, True, 24, 4, 19)]


def _check_margin(masses, what):
    m = torch.cat([x.flatten() for x in masses])
    margin = (m - 1.0).abs().min().item()
    print(f"[sag] {what}: {m.numel()} oracle masses, {(m > 1).double().mean().item():.2f} marked, min |mass - 1| {margin:.2e}")
    assert margin >= 1e-3, "a mass this close to the threshold could flip the mask: pick another seed"


@pytest.mark.parametrize("kind,scale,multi,side,steps,seed", WALKS)
def test_walk_vs_oracle(mini, kind, scale, multi, side, steps, seed):
    from lib.model_zoo.sag import SelfAttentionGuidance
    from oracle import sag_oracle as S
    net, sd, gi = mini
    g = torch.Generator().manual_seed(seed)
    bs, C = 2, 4
    xT = torch.randn(bs, C, side, side, generator=g)
    conds, unconds, okw, ratios = _contexts(gi, g, bs, multi)
    Sm = _sampler(kind, net)
    x_info = {"type": "image", "xt": xT.to(DEV), "sag": SelfAttentionGuidance(0.75)}
    kw = dict(steps=steps, shape=[bs, C, side, side], x_info=x_info, verbose=False, eta=0.)
    cl = _cinfos(conds, unconds, scale, ratios)
    with torch.no_grad():
        x, _ = Sm.sample_multicontext(c_info_list=cl, **kw) if multi else Sm.sample(c_info=cl[0], **kw)
    masses = []
    ref = S.sample(sd, xT, conds, unconds, steps, 0.75, sampler=kind, scale=scale, masses=masses, model_channels=64, **okw)
    what = f"SAG {kind} scale {scale} {'dual' if multi else 'single'} {side}x{side}"
    _check_margin(masses, what)
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=what + " vs oracle")


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_walk_with_inpainting_vs_oracle(mini, kind):
    """one step, so the blend's Philox draws (of later steps) do not enter; the kept region is x0 exactly"""
    from lib.model_zoo.sag import SelfAttentionGuidance
    from oracle import sag_oracle as S
    net, sd, gi = mini
    g = torch.Generator().manual_seed(17)
    bs, C, side = 2, 4, 32
    xT = torch.randn(bs, C, side, side, generator=g)
    x0 = torch.randn(1, C, side, side, generator=g) * 0.8
    lat = torch.zeros(bs, 1, side, side)
    lat[:, :, :, side // 2:] = 1.0
    lat[:, :, :, side // 2 - 1] = 0.5
    conds, unconds, _, _ = _contexts(gi, g, bs, False)
    Sm = _sampler(kind, net)
    x_info = {"type": "image", "xt": xT.to(DEV), "x0": x0.to(DEV), "inpaint_mask": lat.to(DEV), "sag": SelfAttentionGuidance(0.75)}
    with torch.no_grad():
        x, _ = Sm.sample(steps=1, shape=[bs, C, side, side], x_info=x_info, c_info=_cinfo(conds[0], unconds[0], 7.5),
                         verbose=False, eta=0.)
    masses = []
    ref = S.sample(sd, xT, conds, unconds, 1, 0.75, sampler=kind, scale=7.5, x0=x0, mask=lat, masses=masses, model_channels=64,
                   noise_fn=lambda i: torch.zeros(bs, C, side, side))
    _check_margin(masses, f"SAG {kind} with an inpainting mask")
    _cmp(x, ref, cos_min=0.995, tol=0.1, what=f"SAG {kind} with an inpainting mask vs oracle")
    keep = (lat == 0).expand(bs, C, side, side)
    assert torch.equal(x.cpu()[keep], x0.expand(bs, C, side, side)[keep]), "the kept region is x0 exactly"


@pytest.mark.parametrize("kind", ["ddim", "dpmpp"])
def test_graph_equals_eager_and_replays(mini, kind):
    from lib.model_zoo.sag import SelfAttentionGuidance
    net, sd, gi = mini
    g = torch.Generator().manual_seed(29)
    bs, C, side, steps = 2, 4, 32, 5
    xT = torch.randn(bs, C, side, side, generator=g).to(DEV)
    prompts = [(torch.randn(bs, 77, 768, generator=g) * 0.5, torch.randn(bs, 77, 768, generator=g) * 0.5) for _ in range(2)]

    def run(S, p, sag=True):
        x_info = {"type": "image", "xt": xT.clone()}
        if sag:
            x_info["sag"] = SelfAttentionGuidance(0.75)
        with torch.no_grad():
            return S.sample(steps=steps, shape=[bs, C, side, side], x_info=x_info, c_info=_cinfo(p[0], p[1], 7.5), verbose=False,
                            eta=0.)[0]

    Sg, Se, Sp = _sampler(kind, net), _sampler(kind, net, use_cuda_graph=False), _sampler(kind, net)
    assert torch.equal(run(Sg, prompts[0]), run(Se, prompts[0])), "graph and eager SAG walks agree bit for bit"
    graph, launches = next(iter(Sg._graphs.values()))[0], Sg.last_step_launches
    Sg.last_step_launches = None
    second = run(Sg, prompts[1])
    assert next(iter(Sg._graphs.values()))[0] is graph, "the second call replays the cached graph"
    assert Sg.last_step_launches is None, "without an eager step"
    assert torch.equal(second, run(Se, prompts[1])), "the replay on new prompts equals the eager walk"
    run(Sp, prompts[0], sag=False)
    print(f"[sag] {kind} launches per step: unguided {Sp.last_step_launches}, SAG {launches}")
    assert launches > Sp.last_step_launches
