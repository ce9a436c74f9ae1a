"""Pins oracle/pil_resample.py (restatement of Pillow's 8-bit bicubic resampling, the arithmetic behind the reference's
CLIPProcessor host path, clip.py:88-94) BIT-EXACTLY against Pillow itself, and the full CLIP preprocessing restatement
against the product's host path (CLIPImageContextEncoder.preprocess, which calls Pillow)."""
import numpy as np
import pytest
import torch


@pytest.mark.parametrize("h,w,oh,ow", [(37, 53, 17, 24), (300, 420, 224, 313), (512, 512, 224, 224), (100, 64, 350, 224),
                                       (224, 224, 224, 224), (7, 5, 3, 2), (64, 64, 65, 63), (1, 9, 4, 4)])
def test_bicubic_u8_resize_is_bit_exact_with_pillow(h, w, oh, ow):
    from PIL import Image
    from oracle.pil_resample import resize_bicubic_u8
    img = np.random.RandomState(h * 1000 + w).randint(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(img).resize((ow, oh), resample=Image.BICUBIC))
    mine = resize_bicubic_u8(img, ow, oh)
    assert mine.shape == ref.shape
    assert np.array_equal(mine, ref), f"{np.abs(mine.astype(int) - ref.astype(int)).max()} levels off on {(mine != ref).sum()} samples"


def test_clip_preprocess_restatement_matches_the_host_path():
    from lib.model_zoo.clip import CLIPImageContextEncoder
    from oracle.pil_resample import clip_preprocess
    g = torch.Generator().manual_seed(3)
    for shape in ((2, 3, 256, 256), (1, 3, 300, 420), (1, 3, 512, 384)):
        t = torch.rand(*shape, generator=g)
        ref = CLIPImageContextEncoder.preprocess(t)                 # ToPILImage semantics + Pillow resize + crop + normalise
        mine = torch.from_numpy(clip_preprocess(t.numpy()))
        assert mine.shape == ref.shape
        assert (mine - ref).abs().max().item() <= 1e-6


@pytest.mark.parametrize("n_in,n_out", [(300, 224), (420, 313), (512, 224), (64, 350), (9, 4), (224, 224), (37, 17)])
def test_product_coefficient_tables_equal_the_oracle_restatement(n_in, n_out):
    """Two independent writings of Pillow's coefficient computation (product: lib/model_zoo/clip.py, oracle: pil_resample.py)."""
    from lib.model_zoo.clip import CLIPImageContextEncoder
    from oracle.pil_resample import coefficients
    pb, pk = CLIPImageContextEncoder.pil_bicubic_coeffs(n_in, n_out)
    ob, ok = coefficients(n_in, n_out)
    assert np.array_equal(pb, ob) and np.array_equal(pk, ok)
    assert pk.dtype == np.int32 and abs(int(pk.sum(axis=1).max()) - (1 << 22)) <= pk.shape[1]      # weights sum to one


@pytest.mark.parametrize("n_in,n_out", [(2048, 896), (512, 224), (1024, 224), (50, 224), (60, 268), (130, 291), (100, 224)])
def test_resample_accumulator_cannot_overflow_int32(n_in, n_out):
    """vdb_resample_h_u8 / vdb_resample_v_crop_norm accumulate 1 << 21 + sum_t u8 * kk in int32: for the tables of the shapes the
    device preprocessing is tested at (strong downscales with 11 and 21 taps, upscales), 255 * sum |kk| + 2^21 stays below 2^31."""
    from lib.model_zoo.clip import CLIPImageContextEncoder
    _, kk = CLIPImageContextEncoder.pil_bicubic_coeffs(n_in, n_out)
    worst = 255 * int(np.abs(kk.astype(np.int64)).sum(axis=1).max()) + (1 << 21)
    assert worst < 2 ** 31, f"{n_in} -> {n_out}: {worst} >= 2^31"
