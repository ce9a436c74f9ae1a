"""Editing, CPU side (lib/model_zoo/edit.py): the inversion rows against the fp64 oracle, DiffEdit's mask rule on synthetic eps,
the refusals of invert and of sampling from an inversion (all raised before any device work), and the argument checks of the
three C entry points."""
import types

import numpy as np
import pytest
import torch

from oracle import edit_oracle as E
from oracle import vd_oracle as O


def _fake_model():
    sch = O.ddpm_schedule(1000)
    return types.SimpleNamespace(num_timesteps=1000, device="cpu", alphas_cumprod=sch["alphas_cumprod"], betas=sch["betas"],
                                 alphas_cumprod_prev=sch["alphas_cumprod_prev"])


def _cinfo(bs=2, scale=1.0):
    return {"type": "text", "conditioning": torch.zeros(bs, 77, 768), "unconditional_conditioning": torch.zeros(bs, 77, 768),
            "unconditional_guidance_scale": scale}


@pytest.mark.parametrize("steps,k", [(5, 5), (20, 7), (50, 25), (50, 50)])
def test_inversion_rows(steps, k):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.edit import inversion_rows
    S = DDIMSampler(_fake_model())
    S.make_schedule(steps, verbose=False)
    rows = inversion_rows(S.ddim_alphas, S.ddim_alphas_prev, k)
    sched = O.ddim_schedule(O.ddpm_schedule(1000)["alphas_cumprod"], steps)
    want = E.inversion_rows(sched["alphas"], sched["alphas_prev"], k)
    assert rows.dtype == np.float32 and rows.shape == (k, 4)
    assert np.array_equal(rows, want.astype(np.float32))
    assert np.all(rows[:, 2] == 0)
    # the inversion row swaps the forward row's a_t and a_prev: {a_i, a'_i} -> {a'_i, a_i}
    assert np.array_equal(rows[:, 0], np.asarray(S.ddim_alphas_prev, dtype=np.float32)[:k])
    assert np.array_equal(rows[:, 1], np.asarray(S.ddim_alphas, dtype=np.float32)[:k])
    # inversion step i followed by forward step i from the same eps is the identity, up to fp64 rounding
    g = np.random.default_rng(steps)
    x, e = g.standard_normal(64), g.standard_normal(64)
    for i in range(k):
        ap, a = want[i, 0], want[i, 1]
        y = np.sqrt(a) * (x - np.sqrt(1 - ap) * e) / np.sqrt(ap) + np.sqrt(1 - a) * e
        back = np.sqrt(ap) * (y - np.sqrt(1 - a) * e) / np.sqrt(a) + np.sqrt(1 - ap) * e
        assert np.allclose(back, x, rtol=0, atol=1e-12)


def test_mask_rule_on_synthetic_eps():
    g = np.random.default_rng(0)
    D, bs, C, H, W = 4, 2, 4, 16, 16
    e = g.standard_normal((D, bs, C, H, W))
    m, d, cap = E.diffedit_mask(e, e.copy())
    assert m.shape == (bs, 1, H, W) and not m.any() and np.all(cap == 0), "identical sides: all 0"
    region = np.zeros((bs, H, W), dtype=bool)
    region[0, 2:7, 3:9] = True
    region[1, 10:14, 0:16] = True
    tgt = e + 0.01 * g.standard_normal(e.shape)
    tgt += 2.0 * region[None, :, None]
    m, d, cap = E.diffedit_mask(e, tgt)
    assert np.array_equal(m[:, 0] == 1, region), "a planted difference region is exactly the mask"
    # the rule: d >= cap / 2 with cap = 3 mean(d)
    assert np.array_equal(m[:, 0] == 1, d[:, 0] >= 0.5 * cap[:, None, None])


def test_invert_refusals():
    """invert refuses text latents, a wrong batch and an out-of-range k before any device work (the fake model is on the CPU,
    where a call that passed them would raise RuntimeError instead); DPM-Solver++ and PLMS have no inversion."""
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    from lib.model_zoo.plms import PLMSSampler
    S = DDIMSampler(_fake_model())
    with pytest.raises(ValueError, match="text latent"):
        S.invert(5, torch.zeros(2, 768), _cinfo())
    with pytest.raises(ValueError, match="x0"):
        S.invert(5, torch.zeros(3, 4, 8, 8), _cinfo())
    for k in (0, -1, 6):
        with pytest.raises(ValueError, match="k = "):
            S.invert(5, torch.zeros(2, 4, 8, 8), _cinfo(), k=k)
    with pytest.raises(ValueError, match="text latent"):
        S.invert_multicontext(5, torch.zeros(2, 768), [_cinfo(), _cinfo()])
    for x0 in (torch.zeros(2, 4, 8, 8), torch.zeros(1, 4, 8, 8)):
        with pytest.raises(RuntimeError, match="no CPU path"):
            S.invert(5, x0, _cinfo(), k=3)
    for cls in (DPMSolverSampler, PLMSSampler):
        with pytest.raises(NotImplementedError, match="no inversion"):
            cls(_fake_model()).invert(5, torch.zeros(2, 4, 8, 8), _cinfo())
        with pytest.raises(NotImplementedError, match="no inversion"):
            cls(_fake_model()).invert_multicontext(5, torch.zeros(2, 4, 8, 8), [_cinfo()])


def test_mismatched_context_batches_are_refused():
    """diffedit_mask and invert refuse contexts whose batches differ, before any device work (a fake model on the CPU: a call that
    passed the checks would fail on its first device operation instead)."""
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.edit import diffedit_mask
    net = _fake_model()
    x0 = torch.zeros(2, 4, 8, 8)
    two, one = _cinfo(2, 7.5), _cinfo(1, 7.5)
    uncond_one = dict(_cinfo(2, 7.5), unconditional_conditioning=torch.zeros(1, 77, 768))
    for src, tgt, match in ((two, one, "batch of 1, src's 2"), (one, two, "batch of 2, src's 1"),
                            (two, [two, _cinfo(1, 7.5)], "context 1"), ([two, one], two, "context 1"),
                            (two, uncond_one, "unconditional_conditioning")):
        with pytest.raises(ValueError, match=match):
            diffedit_mask(net, x0, src, tgt, steps=10)
    # at scale 1 the unconditional context is never read, so its batch does not matter: the call passes the checks and stops
    # at its first device operation
    with pytest.raises(ValueError, match="need CUDA tensors"):
        diffedit_mask(net, x0, dict(uncond_one, unconditional_guidance_scale=1.0), two, steps=10)
    S = DDIMSampler(net)
    with pytest.raises(ValueError, match="context 1"):
        S.invert_multicontext(5, x0, [_cinfo(2), _cinfo(1)])
    with pytest.raises(ValueError, match="unconditional_conditioning"):
        S.invert(5, x0, uncond_one)


def _inversion(steps=5, k=3, bs=2, H=8, W=8):
    """an Inversion built on the CPU without a device walk (the trajectory's values do not matter to the refusals)"""
    from lib.model_zoo.edit import Inversion
    inv = Inversion.__new__(Inversion)
    inv.trajectory = torch.zeros(k + 1, bs, H, W, 4)
    inv.steps, inv.k, inv.bs, inv.shape = steps, k, bs, (bs, 4, H, W)
    inv.timesteps = O.make_ddim_timesteps(steps)
    inv.xt = torch.zeros(bs, 4, H, W)
    return inv


@pytest.mark.parametrize("multi", [False, True])
def test_sample_from_inversion_refusals(multi):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    from lib.model_zoo.plms import PLMSSampler
    inv = _inversion()
    shape = [2, 4, 8, 8]
    cases = [
        (5, [2, 4, 8, 16], {}, "shape"),
        (5, [1, 4, 8, 8], {}, "shape"),
        (6, shape, {}, "steps=5"),
        (5, shape, {"xt": torch.zeros(2, 4, 8, 8)}, "'xt'"),
        (5, shape, {"x0": torch.zeros(2, 4, 8, 8)}, "'x0'"),
        (5, shape, {"x0_forward_timesteps": 2}, "'x0_forward_timesteps'"),
        (5, shape, {"inpaint_mask": torch.ones(3, 1, 8, 8)}, "inpaint_mask"),
        (5, shape, {"inpaint_mask": torch.full((1, 1, 8, 8), 1.5)}, "\\[0, 1\\]"),
    ]
    for S in (DDIMSampler(_fake_model()), DPMSolverSampler(_fake_model())):
        for steps, shp, extra, match in cases:
            x_info = dict({"type": "image", "inversion": inv}, **extra)
            with pytest.raises(ValueError, match=match):
                if multi:
                    S.sample_multicontext(steps=steps, shape=shp, x_info=x_info, c_info_list=[_cinfo(), _cinfo()], verbose=False)
                else:
                    S.sample(steps=steps, shape=shp, x_info=x_info, c_info=_cinfo(), verbose=False)
        with pytest.raises(ValueError, match="Inversion"):
            S.sample(steps=5, shape=shape, x_info={"type": "image", "inversion": torch.zeros(4)}, c_info=_cinfo(), verbose=False)
        # valid inputs pass the checks and reach the device check
        for mask in (None, torch.rand(2, 1, 8, 8), torch.rand(1, 1, 64, 64)):
            x_info = {"type": "image", "inversion": inv}
            if mask is not None:
                x_info["inpaint_mask"] = mask
            with pytest.raises(RuntimeError, match="no CPU path"):
                S.sample(steps=5, shape=shape, x_info=x_info, c_info=_cinfo(), verbose=False)
    with pytest.raises(NotImplementedError, match="inversion"):
        PLMSSampler(_fake_model()).sample(steps=5, shape=shape, x_info={"type": "image", "inversion": inv}, c_info=_cinfo(),
                                          verbose=False)


def test_a_walk_from_an_inversion_draws_nothing():
    """no Philox key is drawn for the trajectory blend: torch's generator is untouched by a masked walk from an inversion"""
    from lib.model_zoo.ddim import DDIMSampler
    S = DDIMSampler(_fake_model())
    torch.manual_seed(0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        S.sample(steps=5, shape=[2, 4, 8, 8], x_info={"type": "image", "inversion": _inversion(), "inpaint_mask": torch.ones(1, 1, 8, 8)},
                 c_info=_cinfo(), verbose=False)
    after = torch.randint(0, 2 ** 62, (1,)).item()
    torch.manual_seed(0)
    assert after == torch.randint(0, 2 ** 62, (1,)).item()


def test_entry_points_reject_bad_arguments_without_gpu():
    """vdb_latent_store_slot_f32, vdb_inversion_blend_f32 and vdb_diffedit_mask_f32 refuse null, misaligned, empty and overlapping
    arguments before any launch (the fake addresses below are never dereferenced: every call fails its checks)."""
    from vdb200._lib import lib
    before = lib.vdb_launch_count()
    n, slots = 512, 6
    st = dict(x=0x100000, ring=0x200000, slots=slots, idx=0x600000, off=1, n=n)

    def store(**kw):
        a = dict(st, **kw)
        return lib.vdb_latent_store_slot_f32(a["x"], a["ring"], a["slots"], a["idx"], a["off"], a["n"], None)

    for k in ("x", "ring", "idx"):
        assert store(**{k: None}) == 1 and b"latent_store_slot: null" in lib.vdb_last_error(), k
    for k, v in (("n", 0), ("n", -4), ("slots", 0), ("slots", -1)):
        assert store(**{k: v}) == 1 and b"empty" in lib.vdb_last_error(), (k, v)
    for k in ("x", "ring"):
        assert store(**{k: st[k] + 4}) == 1 and b"16-byte aligned" in lib.vdb_last_error(), k
    for addr in (0x200000, 0x200000 + 4 * (slots * n - 4), 0x200000 - 4 * (n - 4)):
        assert store(x=addr) == 1 and b"overlaps" in lib.vdb_last_error(), addr

    bs, hw, c = 2, 64, 4
    nb = bs * hw * c
    ok = dict(x=0x100000, dup=0x180000, ring=0x200000, slots=slots, mask=0x400000, per=1, idx=0x600000, bs=bs, hw=hw, c=c)

    def blend(**kw):
        a = dict(ok, **kw)
        return lib.vdb_inversion_blend_f32(a["x"], a["dup"], a["ring"], a["slots"], a["mask"], a["per"], a["idx"], a["bs"],
                                           a["hw"], a["c"], None)

    for k in ("x", "ring", "mask", "idx"):
        assert blend(**{k: None}) == 1 and b"inversion_blend: null" in lib.vdb_last_error(), k
    for k in ("slots", "bs", "hw", "c"):
        for v in (0, -4):
            assert blend(**{k: v}) == 1 and b"empty" in lib.vdb_last_error(), (k, v)
    for k in ("x", "dup", "ring", "mask"):
        assert blend(**{k: ok[k] + 4}) == 1 and b"16-byte aligned" in lib.vdb_last_error(), k
    for out in ("x", "dup"):
        o = ok[out]
        for k, length in (("ring", slots * nb), ("mask", bs * hw)):
            for addr in (o, o + 4 * (nb - 4), o - 4 * (length - 4)):
                assert blend(**{k: addr}) == 1 and b"overlaps" in lib.vdb_last_error(), (out, k, addr)
    # the mask's extent follows mask_per_item
    assert blend(per=1, mask=ok["x"] - 4 * hw) == 1 and b"overlaps" in lib.vdb_last_error()

    D = 3
    ne = D * bs * hw * c
    mk = dict(su=0x100000, sc=0x200000, tu=0x300000, tc=0x400000, D=D, bs=bs, hw=hw, c=c, ratio=3.0, out=0x500000)

    def mask(**kw):
        a = dict(mk, **kw)
        return lib.vdb_diffedit_mask_f32(a["su"], a["sc"], 7.5, a["tu"], a["tc"], 5.0, a["D"], a["bs"], a["hw"], a["c"], a["ratio"],
                                         a["out"], None)

    for k in ("sc", "tc", "out"):
        assert mask(**{k: None}) == 1 and b"diffedit_mask: null" in lib.vdb_last_error(), k
    for k in ("D", "bs", "hw", "c"):
        for v in (0, -2):
            assert mask(**{k: v}) == 1 and b"empty" in lib.vdb_last_error(), (k, v)
    for v in (0.0, -1.0, float("nan"), float("inf")):
        assert mask(ratio=v) == 1 and b"ratio" in lib.vdb_last_error(), v
    for k in ("su", "sc", "tu", "tc", "out"):
        assert mask(**{k: mk[k] + 4}) == 1 and b"16-byte aligned" in lib.vdb_last_error(), k
    for k in ("su", "sc", "tu", "tc"):
        for addr in (mk[k], mk[k] + 4 * (ne - 4), mk[k] - 4 * (bs * hw - 4)):
            assert mask(out=addr) == 1 and b"overlaps" in lib.vdb_last_error(), (k, addr)
    assert lib.vdb_launch_count() == before
