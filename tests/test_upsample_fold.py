"""Folding "nearest-2x upsample + 3x3 conv" into four 2x2-tap convs on the source image: the weight folding and the tap /
parity conventions handed to the kernel (conv modes 7..10 of vdb_conv3x3_bf16, each storing one parity of the interleaved
result) are checked here on the CPU against torch's own upsample + conv2d (reference semantics:
openaimodel.py:107-117, autokl_modules.py:54-58).  The emulation below consumes the folded weights exactly as the kernel
does: K ordered (ty, tx, ci), source pixel (y + ty - 1 + py, x + tx - 1 + px), zero fill outside the image."""
import pytest
import torch
import torch.nn.functional as F


def emulate_kernel(x, wf, bias):
    """x [B,C,H,W] fp32, wf [4, N, 4*C] (any float dtype) -> [B,N,2H,2W], mirroring modes 7..10."""
    B, C, H, W = x.shape
    N = wf.shape[1]
    xp = F.pad(x, (1, 1, 1, 1))                         # TMA zero-fills out-of-image source pixels
    out = torch.zeros(B, N, 2 * H, 2 * W)
    for par in range(4):
        py, px = par >> 1, par & 1
        acc = torch.zeros(B, N, H, W)
        for t in range(4):
            ty, tx = t >> 1, t & 1
            dh, dw = ty - 1 + py, tx - 1 + px           # ASeg{dw, dh} of igemm.cu
            src = xp[:, :, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W]
            wt = wf[par].float()[:, t * C:(t + 1) * C]  # [N, C]
            acc += torch.einsum("bchw,nc->bnhw", src, wt)
        out[:, :, py::2, px::2] = acc + bias[None, :, None, None]     # out[b, 2y+py, 2x+px]
    return out


@pytest.mark.parametrize("B,C,N,H,W", [(2, 8, 6, 5, 7), (1, 16, 16, 8, 8), (1, 4, 3, 1, 1), (2, 8, 8, 2, 3)])
def test_folded_weights_reproduce_upsample_then_conv(B, C, N, H, W):
    from lib.model_zoo.diffusion_utils import fold_upsample_conv3x3
    g = torch.Generator().manual_seed(B * 100 + C)
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(N, C, 3, 3, generator=g) * 0.2
    b = torch.randn(N, generator=g)
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, b, padding=1)
    # exact in fp32 (the folding only re-associates sums) ...
    from lib.model_zoo import diffusion_utils as du
    wf = du.fold_upsample_conv3x3(w)                    # bf16, as shipped to the kernel
    assert wf.shape == (4, N, 4 * C) and wf.dtype == torch.bfloat16
    out = emulate_kernel(x, wf, b)
    # ... and within bf16 weight rounding of the folded copy
    assert (out - ref).abs().max() <= 2e-2 * ref.abs().max() + 1e-3
    # fp32 folding (no bf16 rounding) must match to round-off: this is the check of the conventions themselves
    groups = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    wf_exact = torch.stack([torch.stack([sum(w[:, :, ky, kx] for ky in groups[par >> 1][t >> 1] for kx in groups[par & 1][t & 1])
                                         for t in range(4)], dim=1).reshape(N, -1) for par in range(4)])
    assert (emulate_kernel(x, wf_exact, b) - ref).abs().max() <= 1e-4 * (1 + ref.abs().max())
    assert (wf.float() - wf_exact).abs().max() <= 8e-3 * wf_exact.abs().max() + 1e-6


def test_fold_rule():
    """fold where the source grid fills the machine (>= 2048 pixels) and the output channels suit the interleaved TMA store"""
    from lib.model_zoo.diffusion_utils import upsample_fold_enabled
    assert upsample_fold_enabled(4096, 320) and upsample_fold_enabled(2048, 32)
    assert not upsample_fold_enabled(512, 320) and not upsample_fold_enabled(2047, 320)
    assert not upsample_fold_enabled(4096, 48) and not upsample_fold_enabled(1 << 20, 3)
