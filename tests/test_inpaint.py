"""Inpainting, CPU side (lib/model_zoo/inpaint.py): the blend table, mask resolution and input refusals of the samplers, the
argument checks of the C entry points, and the oracle's masked walk (oracle/inpaint_oracle.py) on the analytic Gaussian model
against its closed form."""
import types

import numpy as np
import pytest
import torch

from oracle import dpm_solver_oracle as D
from oracle import inpaint_oracle as I
from oracle import vd_oracle as O

AC = O.ddpm_schedule(1000)["alphas_cumprod"]
MU, S = 0.3, 1.0


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


@pytest.mark.parametrize("steps", [5, 20, 50])
def test_blend_table_rows(steps):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.inpaint import blend_table
    S = DDIMSampler(_fake_model())
    S.make_schedule(steps, verbose=False)
    t = blend_table(S.ddim_alphas_prev)
    assert t.dtype == np.float32 and t.shape == (len(S.ddim_timesteps), 2)
    assert t[0, 0] == 1.0 and t[0, 1] == 0.0
    a = np.asarray(S.ddim_alphas_prev, dtype=np.float64)[1:]
    assert np.array_equal(t[1:, 0], np.sqrt(a).astype(np.float32))
    assert np.array_equal(t[1:, 1], np.sqrt(1.0 - a).astype(np.float32))
    # the targets are the grid's previous points: the oracle's rows, rounded to fp32
    assert np.array_equal(t, I.blend_rows(AC, S.ddim_timesteps).astype(np.float32))


def test_mask_resolution():
    from lib.model_zoo.inpaint import mask_resolution
    assert mask_resolution((4, 1, 64, 64), 4, 64, 64) == "latent"
    assert mask_resolution((1, 1, 64, 64), 4, 64, 64) == "latent"
    assert mask_resolution((4, 1, 512, 512), 4, 64, 64) == "pixel"
    assert mask_resolution((1, 1, 256, 128), 2, 32, 16) == "pixel"
    for bad in ((2, 1, 64, 64), (4, 4, 64, 64), (4, 64, 64), (4, 1, 64, 32), (4, 1, 128, 128), (4, 1, 511, 512), (1, 64, 64)):
        with pytest.raises(ValueError, match="inpaint_mask"):
            mask_resolution(bad, 4, 64, 64)


def _cinfo():
    return {"type": "text", "conditioning": torch.zeros(1, 77, 768), "unconditional_conditioning": torch.zeros(1, 77, 768),
            "unconditional_guidance_scale": 7.5}


def _samplers():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    return [DDIMSampler(_fake_model()), DPMSolverSampler(_fake_model())]


@pytest.mark.parametrize("multi", [False, True])
def test_sampler_refusals(multi):
    """Every refusal is raised before any device work (the fake model is on the CPU, where a call that passed them would raise
    RuntimeError instead)."""
    bs, H, W = 2, 8, 8
    x0 = torch.zeros(bs, 4, H, W)
    m = torch.ones(1, 1, H, W)
    cases = [
        ([bs, 768], {"type": "text", "x0": torch.zeros(bs, 768), "inpaint_mask": torch.ones(bs, 768)}, "text latent"),
        ([bs, 4, H, W], {"type": "image", "inpaint_mask": m}, "needs x_info\\['x0'\\]"),
        ([bs, 4, H, W], {"type": "image", "x0": torch.zeros(3, 4, H, W), "inpaint_mask": m}, "x0"),
        ([bs, 4, H, W], {"type": "image", "x0": torch.zeros(bs, 3, H, W), "inpaint_mask": m}, "x0"),
        ([bs, 4, H, W], {"type": "image", "x0": torch.zeros(bs, 4, 2 * H, 2 * W), "inpaint_mask": m}, "x0"),
        ([bs, 4, H, W], {"type": "image", "x0": x0, "inpaint_mask": torch.ones(3, 1, H, W)}, "inpaint_mask"),
        ([bs, 4, H, W], {"type": "image", "x0": x0, "inpaint_mask": torch.ones(bs, 1, 4 * H, 4 * W)}, "inpaint_mask"),
        ([bs, 4, H, W], {"type": "image", "x0": x0, "inpaint_mask": torch.ones(bs, H, W)}, "inpaint_mask"),
        ([bs, 4, H, W], {"type": "image", "x0": x0, "inpaint_mask": torch.full((1, 1, H, W), 1.5)}, "\\[0, 1\\]"),
        ([bs, 4, H, W], {"type": "image", "x0": x0, "inpaint_mask": torch.full((1, 1, H, W), float("nan"))}, "\\[0, 1\\]"),
    ]
    for S in _samplers():
        for shape, x_info, match in cases:
            with pytest.raises(ValueError, match=match):
                if multi:
                    S.sample_multicontext(steps=5, shape=shape, x_info=x_info, c_info_list=[_cinfo(), _cinfo()], verbose=False)
                else:
                    S.sample(steps=5, shape=shape, x_info=x_info, c_info=_cinfo(), verbose=False)
        # valid inputs at both resolutions pass the checks and reach the device check
        for mask in (torch.rand(bs, 1, H, W), torch.rand(1, 1, 8 * H, 8 * W)):
            with pytest.raises(RuntimeError, match="no CPU path"):
                S.sample(steps=5, shape=[bs, 4, H, W], x_info={"type": "image", "x0": x0[:1], "inpaint_mask": mask},
                         c_info=_cinfo(), verbose=False)


def test_key_is_drawn_only_with_a_mask():
    """The Philox key comes from torch's CPU generator, and only when a mask is given."""
    from lib.model_zoo.ddim import DDIMSampler
    S = DDIMSampler(_fake_model())
    for x_info, draws in (({"type": "image"}, 0), ({"type": "image", "x0": torch.zeros(1, 4, 8, 8),
                                                    "inpaint_mask": torch.ones(1, 1, 8, 8)}, 1)):
        torch.manual_seed(0)
        with pytest.raises(RuntimeError, match="no CPU path"):
            S.sample(steps=5, shape=[1, 4, 8, 8], x_info=x_info, c_info=_cinfo(), verbose=False)
        after = torch.randint(0, 2 ** 62, (1,)).item()
        torch.manual_seed(0)
        for _ in range(draws):
            torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)
        assert after == torch.randint(0, 2 ** 62, (1,)).item(), draws


def test_plms_refuses_a_mask():
    from lib.model_zoo.plms import PLMSSampler
    S = PLMSSampler(_fake_model())
    with pytest.raises(NotImplementedError, match="inpainting"):
        S.sample(steps=5, shape=[1, 4, 8, 8], x_info={"type": "image", "x0": torch.zeros(1, 4, 8, 8),
                                                      "inpaint_mask": torch.ones(1, 1, 8, 8)}, c_info=_cinfo(), verbose=False)
    with pytest.raises(NotImplementedError):
        S.sample_multicontext(steps=5, shape=[1, 4, 8, 8], x_info={"type": "image", "inpaint_mask": torch.ones(1, 1, 8, 8)},
                              c_info_list=[_cinfo()], verbose=False)


def test_entry_points_reject_bad_arguments_without_gpu():
    """vdb_inpaint_blend_f32, vdb_inpaint_noise_f32, vdb_mask_to_latent and vdb_composite_f32 refuse null, misaligned, empty and
    overlapping arguments before any launch (the fake addresses below are never dereferenced: every call fails its checks)."""
    from vdb200._lib import lib
    bs, hw, c = 2, 64, 4
    n = bs * hw * c
    ok = dict(x=0x100000, dup=0x200000, x0=0x300000, mask=0x400000, per=1, table=0x500000, idx=0x600000, seed=0x700000,
              noise=0x800000, bs=bs, hw=hw, c=c)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.vdb_inpaint_blend_f32(a["x"], a["dup"], a["x0"], a["mask"], a["per"], a["table"], a["idx"], a["seed"],
                                         a["noise"], a["bs"], a["hw"], a["c"], None)

    before = lib.vdb_launch_count()
    for k in ("x", "x0", "mask", "table", "idx"):
        assert call(**{k: None}) == 1, k
        assert b"inpaint_blend: null" in lib.vdb_last_error()
    assert call(seed=None, noise=None) == 1 and b"null" in lib.vdb_last_error()
    for k in ("bs", "hw", "c"):
        for v in (0, -4):
            assert call(**{k: v}) == 1 and b"empty" in lib.vdb_last_error(), (k, v)
    for k in ("x", "dup", "x0", "mask", "table", "noise"):
        assert call(**{k: ok[k] + 4}) == 1, k
        assert b"16-byte aligned" in lib.vdb_last_error()
    # x0 (n floats), the mask (bs*hw, or hw when broadcast) and the noise (n) against x and x_dup: first and last shared float
    for out in ("x", "dup"):
        o = ok[out]
        for k, length in (("x0", n), ("mask", bs * hw), ("noise", n)):
            for addr in (o, o + 4 * (n - 4), o - 4 * (length - 4)):
                assert call(**{k: addr}) == 1, (out, k, addr)
                assert b"overlaps" in lib.vdb_last_error()
    # the mask's extent follows mask_per_item: a per-item mask of bs*hw floats starting hw floats below x reaches into it
    assert call(per=1, mask=ok["x"] - 4 * hw) == 1 and b"overlaps" in lib.vdb_last_error()
    assert lib.vdb_inpaint_noise_f32(None, 0x600000, 16, 0x100000, None) == 1
    assert lib.vdb_inpaint_noise_f32(0x700000, None, 16, 0x100000, None) == 1
    assert lib.vdb_inpaint_noise_f32(0x700000, 0x600000, 16, None, None) == 1
    assert lib.vdb_inpaint_noise_f32(0x700000, 0x600000, 0, 0x100000, None) == 1 and b"inpaint_noise" in lib.vdb_last_error()
    assert lib.vdb_mask_to_latent(None, 1, 64, 64, 0x100000, None) == 1
    assert lib.vdb_mask_to_latent(0x100000, 0, 64, 64, 0x200000, None) == 1
    for h8, w8 in ((60, 64), (64, 12), (0, 64)):
        assert lib.vdb_mask_to_latent(0x100000, 1, h8, w8, 0x200000, None) == 1 and b"mask_to_latent" in lib.vdb_last_error()
    for k in range(4):
        ptrs = [0x100000, 0x200000, 0x300000, 0x400000]
        ptrs[k] = None
        assert lib.vdb_composite_f32(ptrs[0], ptrs[1], ptrs[2], 1, 2, 3, 64, ptrs[3], None) == 1, k
        assert b"composite: null" in lib.vdb_last_error()
    assert lib.vdb_composite_f32(0x100000, 0x200000, 0x300000, 1, 2, 0, 64, 0x400000, None) == 1
    assert lib.vdb_launch_count() == before


# ---- the oracle's masked walk on the analytic Gaussian model: data N(MU, S^2) independently per element --------------------------
def _setup(steps, n=4000, seed=0):
    ts = O.make_ddim_timesteps(steps)
    g = np.random.default_rng(seed)
    alpha, sigma = D.coefficients(AC, ts)[:2]
    x_T = MU * alpha[-1] + np.sqrt(alpha[-1] ** 2 * S * S + sigma[-1] ** 2) * g.standard_normal(n)
    x0 = MU + S * g.standard_normal(n)
    zs = g.standard_normal((len(ts), n))
    eps = lambda x, i: D.gaussian_eps(x, alpha[i], sigma[i], MU, S)
    return ts, x_T, x0, zs, eps


@pytest.mark.parametrize("order", [1, 2, 3])
def test_oracle_walk_on_the_analytic_model(order):
    steps = 50
    ts, x_T, x0, zs, eps = _setup(steps)
    n = x_T.shape[0]
    alpha, sigma = D.coefficients(AC, ts)[:2]
    a0 = float(AC[0])
    exact = D.gaussian_exact(x_T, alpha[-1], sigma[-1], np.sqrt(a0), np.sqrt(1 - a0), MU, S)
    unmasked = D.walk(x_T, eps, AC.numpy(), ts, order)
    # all generated: the unmasked walk, bit for bit, and the probability-flow solution within the solver's error
    ones = I.dpm_walk(x_T, eps, AC.numpy(), ts, order, x0, np.ones(n), lambda i: zs[i])
    assert np.array_equal(ones, unmasked)
    assert np.abs(ones - exact).max() <= {1: 0.11, 2: 0.05, 3: 0.03}[order]
    # a hard mask: the elements are independent under this model, so the generated ones follow the unmasked walk exactly and
    # the kept ones end at x0 exactly; after step i > 0 a kept element is x0 re-noised to the step's target
    m = (np.arange(n) % 3 != 0).astype(np.float64)
    trace = []
    x_start = I.start(x_T, x0, m, AC.numpy(), int(ts[-1]))
    a_top = float(AC[int(ts[-1])])
    assert np.array_equal(x_start[m == 0], np.sqrt(a_top) * x0[m == 0] + np.sqrt(1 - a_top) * x_T[m == 0])
    out = I.dpm_walk(x_start, eps, AC.numpy(), ts, order, x0, m, lambda i: zs[i], trace=trace)
    assert np.array_equal(out[m == 1], unmasked[m == 1])
    assert np.array_equal(out[m == 0], x0[m == 0])
    rows = I.blend_rows(AC, ts)
    for k, i in enumerate(range(len(ts) - 1, 0, -1)):
        a_to = float(AC[int(ts[i - 1])])
        kept = trace[k][m == 0]
        assert np.allclose(kept, np.sqrt(a_to) * x0[m == 0] + np.sqrt(1 - a_to) * zs[i][m == 0], rtol=0, atol=1e-12)
        assert np.allclose(rows[i], (np.sqrt(a_to), np.sqrt(1 - a_to)), rtol=0, atol=1e-15)
        # x0 ~ N(MU, S^2) re-noised: the forward marginal N(alpha' MU, alpha'^2 S^2 + sigma'^2) at the target point
        mean, var = np.sqrt(a_to) * MU, a_to * S * S + (1 - a_to)
        assert abs(kept.mean() - mean) <= 5 * np.sqrt(var / kept.size)
        assert abs(kept.var() / var - 1) <= 5 * np.sqrt(2.0 / kept.size)


def test_oracle_soft_mask_is_the_convex_mix_at_every_step():
    """A uniform soft mask m: each step's result is m x' + (1 - m) k of the unblended step from the same x."""
    steps = 20
    ts, x_T, x0, zs, eps = _setup(steps, n=500, seed=3)
    m = np.full(x_T.shape, 0.25)
    trace = []
    I.dpm_walk(x_T, eps, AC.numpy(), ts, 1, x0, m, lambda i: zs[i], trace=trace)
    rows = I.blend_rows(AC, ts)
    x = x_T
    for k, i in enumerate(range(len(ts) - 1, -1, -1)):
        tr = []
        D.walk(x, eps, AC.numpy(), ts[:i + 1], 1, trace=tr)      # its first step is the order-1 step from grid point i
        want = 0.25 * tr[0][2] + 0.75 * (rows[i, 0] * x0 + rows[i, 1] * zs[i])
        assert np.allclose(trace[k], want, rtol=0, atol=1e-12), (k, i)
        x = trace[k]
