"""Self-attention guidance, CPU side (lib/model_zoo/sag.py): the combination matrix with 'sag' added to every subset of the
optional inputs, for every sampler and entry point; the argument checks of SelfAttentionGuidance; the oracle's blur taps, nearest
index and mid-map size; and the host-side refusals of the three entry points through the C ABI.  Nothing here touches a device."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_edit import _fake_model
from test_sampler_modes import NO_CPU, SUBSETS, _call, _draws_after, _inputs, expected


def expected_with_sag(sampler, entry, given, text):
    """-> (exception type, message substring, draws) of a call given `given` and 'sag'.  The entry points check their own rows first
    ('sag' is the last entry of each); among the modes SAG checks first."""
    if entry == "p_sample":
        if sampler == "dpm":
            return NotImplementedError, "no single-step form", 0
        r = expected(sampler, entry, given, text)
        return r if r != NO_CPU + (0,) else (NotImplementedError, "self-attention guidance runs inside the sampler's walk", 0)
    if sampler == "plms":
        r = expected(sampler, entry, given, text)
        return r if r != NO_CPU + (0,) else (NotImplementedError, "PLMSSampler has no self-attention guidance", 0)
    if "windows" in given:
        return NotImplementedError, "SAG with windows", 0
    if "prompt_edit" in given:
        return NotImplementedError, "SAG with prompt_edit", 0
    if text:
        return ValueError, "SAG needs an image latent", 0
    return expected(sampler, entry, given, text)


def _sampler(sampler):
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    from lib.model_zoo.plms import PLMSSampler
    return {"ddim": DDIMSampler, "dpm": DPMSolverSampler, "plms": PLMSSampler}[sampler](_fake_model())


@pytest.mark.parametrize("text", [False, True], ids=["image", "text"])
@pytest.mark.parametrize("entry", ["sample", "sample_multicontext", "p_sample"])
@pytest.mark.parametrize("sampler", ["ddim", "dpm", "plms"])
def test_combination_matrix_with_sag(sampler, entry, text):
    from lib.model_zoo.sag import SelfAttentionGuidance
    states = [_draws_after(n) for n in range(3)]
    for given in [s for s in SUBSETS if not {"regions", "sag"} & set(s)]:      # 'sag' is added to each below
        exc, match, draws = expected_with_sag(sampler, entry, given, text)
        shape, x_info, c_infos = _inputs(given, text)
        x_info["sag"] = SelfAttentionGuidance(0.75)
        S = _sampler(sampler)
        torch.manual_seed(0)
        with pytest.raises(exc) as info:
            _call(S, entry, shape, x_info, c_infos)
        assert match in str(info.value), (given, str(info.value))
        assert torch.equal(torch.get_rng_state(), states[draws]), (given, draws)


@pytest.mark.parametrize("sampler", ["ddim", "dpm"])
def test_regions_and_small_latents_are_refused(sampler):
    from lib.model_zoo.regions import Region, Regions
    from lib.model_zoo.sag import SelfAttentionGuidance
    shape, x_info, c_infos = _inputs((), False)
    x_info.update(sag=SelfAttentionGuidance(), regions=Regions([Region(torch.ones(1, 8, 8), torch.zeros(2, 77, 768))]))
    with pytest.raises(NotImplementedError, match="SAG with regions"):
        _call(_sampler(sampler), "sample", shape, x_info, c_infos)
    for side in ((4, 8), (8, 4)):
        shape = [2, 4, *side]
        x_info = {"type": "image", "sag": SelfAttentionGuidance()}
        with pytest.raises(ValueError, match="latent sides must be >= 5"):
            _call(_sampler(sampler), "sample", shape, x_info, c_infos)
    x_info = {"type": "image", "sag": 0.75}
    with pytest.raises(ValueError, match="must be a sag.SelfAttentionGuidance"):
        _call(_sampler(sampler), "sample", [2, 4, 8, 8], x_info, c_infos)


def test_scale_checks():
    from lib.model_zoo.sag import SelfAttentionGuidance
    assert SelfAttentionGuidance().scale == 0.75
    for ok in (1, 0.1, np.float32(2.5), 100.0):
        assert SelfAttentionGuidance(ok).scale == float(ok)
    for bad in (0, 0.0, -0.5, float("nan"), float("inf"), -float("inf"), None, "big", [1.0]):
        with pytest.raises(ValueError, match="SelfAttentionGuidance: scale"):
            SelfAttentionGuidance(bad)


def test_oracle_blur_taps_follow_the_formula():
    from oracle import sag_oracle as S
    g = S.taps()
    assert g.shape == (9,) and math.isclose(g.sum(), 1.0, rel_tol=0, abs_tol=1e-15)
    for k in range(-4, 5):
        assert math.isclose(g[k + 4] / g[4], math.exp(-0.5 * k * k), rel_tol=1e-14)
    x = torch.randn(2, 4, 11, 13, dtype=torch.float64)
    # the 2-D kernel is the outer product: blurring equals a separable pass along each axis, and a constant stays constant
    gt = torch.from_numpy(g)
    rows = F.conv2d(F.pad(x, (4, 4, 0, 0), mode="reflect"), gt.view(1, 1, 1, 9).expand(4, 1, 1, 9).contiguous(), groups=4)
    sep = F.conv2d(F.pad(rows, (0, 0, 4, 4), mode="reflect"), gt.view(1, 1, 9, 1).expand(4, 1, 9, 1).contiguous(), groups=4)
    assert torch.allclose(S.blur(x), sep, rtol=0, atol=1e-13)
    assert torch.allclose(S.blur(torch.full((1, 1, 6, 5), 3.0, dtype=torch.float64)), torch.tensor(3.0, dtype=torch.float64))


@pytest.mark.parametrize("n_out,n_in", [(64, 8), (40, 5), (48, 6), (32, 4), (24, 3), (17, 3), (5, 1), (100, 13)])
def test_nearest_index_matches_interpolate(n_out, n_in):
    from oracle import sag_oracle as S
    src = torch.arange(n_in, dtype=torch.float64).view(1, 1, n_in, 1)
    want = F.interpolate(src, size=(n_out, 1), mode="nearest").view(-1).long().numpy()
    assert np.array_equal(S.nearest_index(n_out, n_in), want)


def test_mid_map_size_is_three_ceiling_halvings_of_the_layout():
    from lib.model_zoo.sag import MID_DOWNSAMPLES, mid_size
    from oracle import sag_oracle as S
    from oracle import vd_oracle as O
    assert S.mid_block(O.unet_layout())[1] == MID_DOWNSAMPLES == 3
    for H, W in ((64, 64), (40, 48), (5, 6), (96, 128), (33, 17), (24, 24), (512, 512)):
        want = F.conv2d(torch.zeros(1, 1, H, W), torch.zeros(1, 1, 3, 3), stride=2, padding=1)
        for _ in range(2):
            want = F.conv2d(want, torch.zeros(1, 1, 3, 3), stride=2, padding=1)
        assert mid_size(H, W) == S.mid_size(H, W) == tuple(want.shape[2:]), (H, W)
    assert mid_size(64, 64) == (8, 8)


def test_entry_points_reject_bad_arguments_without_gpu():
    """vdb_sattn_key_mass_f32, vdb_sag_degrade_f32 and vdb_sag_guide_f32 refuse bad arguments before any launch (the fake addresses
    are never dereferenced)."""
    from vdb200._lib import lib
    before = lib.vdb_launch_count()
    err = lambda: lib.vdb_last_error()

    km = dict(q=0x100000, k=0x100000, ldq=2 * 8 * 192, ldk=2 * 8 * 192, qc=0, kc=8 * 192, st=0x800000, mass=0x900000, n=2, row0=0,
              H=8, N=64, kv=0, d=160)

    def mass(**kw):
        a = dict(km, **kw)
        return lib.vdb_sattn_key_mass_f32(a["q"], a["ldq"], a["qc"], a["k"], a["ldk"], a["kc"], a["st"], 0.125, a["mass"], a["n"],
                                          a["row0"], a["H"], a["N"], a["kv"], a["d"], 0.08, None)

    for k in ("q", "k", "st", "mass"):
        assert mass(**{k: None}) == 1 and b"sattn_key_mass: null" in err(), k
    for k in ("n", "H", "N"):
        assert mass(**{k: 0}) == 1 and b"sattn_key_mass: null" in err(), k
    assert mass(row0=-1) == 1 and b"null/empty" in err()
    assert mass(N=4097) == 3 and b"at most 4096 tokens" in err()
    for d in (168, 44, 0):
        assert mass(d=d) == 3 and b"d_head" in err(), d
    assert mass(kv=40) == 1 and b"kv_bstride >= N" in err()
    assert mass(kc=8 * 192 + 1) == 1 and b"even column offsets" in err()
    assert mass(ldk=8 * 192 * 2 - 2) == 1 and b"ldq, ldk >= col0" in err()
    assert mass(ldq=2 * 8 * 192 + 1) == 1 and b"even ldq" in err()
    assert mass(mass=0x900002) == 1 and b"4-byte aligned" in err()
    assert mass(st=0x900000 + 4 * 64) == 1 and b"mass overlaps stats" in err()

    dg = dict(x=0x100000, e=0x200000, mass=0x300000, tab=0x400000, idx=0x500000, bs=2, H=64, W=64, C=4, hm=8, wm=8, out=0x600000)

    def degrade(**kw):
        a = dict(dg, **kw)
        return lib.vdb_sag_degrade_f32(a["x"], a["e"], a["mass"], a["tab"], a["idx"], a["bs"], a["H"], a["W"], a["C"], a["hm"], a["wm"],
                                       a["out"], None)

    for k in ("x", "e", "mass", "tab", "idx", "out"):
        assert degrade(**{k: None}) == 1 and b"sag_degrade: null" in err(), k
    for k in ("bs", "H", "W", "C", "hm", "wm"):
        assert degrade(**{k: 0}) == 1 and b"sag_degrade: null" in err(), k
    for H, W in ((4, 64), (64, 4)):
        assert degrade(H=H, W=W, hm=1, wm=1) == 1 and b"reflect padding" in err(), (H, W)
    assert degrade(C=9) == 3 and b"C <= 8" in err()
    assert degrade(hm=65) == 3 and b"hm <= H" in err()
    assert degrade(H=128, W=128, hm=65, wm=65) == 3 and b"hm * wm <= 4096" in err()
    for k in ("x", "e", "mass", "tab", "idx", "out"):
        assert degrade(**{k: dg[k] + 2}) == 1 and b"4-byte aligned" in err(), k
    for k in ("x", "e", "mass"):
        assert degrade(out=dg[k] + 4) == 1 and b"out overlaps" in err(), k

    def guide(eu=0x100000, ec=0x200000, ed=0x300000, s=0.75, n=1024):
        return lib.vdb_sag_guide_f32(eu, ec, ed, s, n, None)

    for kw in (dict(ec=None), dict(ed=None), dict(n=0)):
        assert guide(**kw) == 1 and b"sag_guide: null" in err(), kw
    for s in (float("nan"), float("inf")):
        assert guide(s=s) == 1 and b"finite" in err()
    for kw in (dict(eu=0x100002), dict(ec=0x200001), dict(ed=0x300002)):
        assert guide(**kw) == 1 and b"4-byte aligned" in err(), kw
    for kw in (dict(ed=0x200000 + 4), dict(eu=0x300000 - 4), dict(eu=0x200000)):
        assert guide(**kw) == 1 and b"must not overlap" in err(), kw
    assert lib.vdb_launch_count() == before, "no refusal launches a kernel"
