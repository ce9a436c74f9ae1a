"""Semantic/style disentanglement on the GPU (vdb_rank_adjust_f32): accuracy against the fp64 oracle with tolerances anchored to the
reference's own fp32 rounding, batching, fp16, the default Gaussian start, CUDA-graph capture, and the image-context path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
LVLS = (0.0, 0.1, 0.25, 0.4, 0.6, 0.75, 0.9, 1.0)


def inputs(m):
    """The golden's Gaussian and gapped inputs (regenerated from their seed); m = 257 puts a global token in front, as when disentanglement_noglobal is False."""
    from oracle.disentangle_oracle import golden_inputs
    x = torch.cat(golden_inputs())
    if m == 257:
        g = torch.Generator().manual_seed(8)
        x = torch.cat([x[:, :1] + 0.5 * torch.randn(2, 1, 768, generator=g), x], dim=1)
    return [x[i:i + 1] for i in range(2)]


def start(m, seed=5):
    return torch.randn(m, 20, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("m", [256, 257])
def test_accuracy_against_fp64_oracle(m):
    """Max |product - fp64| <= 4 x the reference's own fp32 error + 1e-6 std(x), per input and lvl; S to 1e-5 relative."""
    from lib.model_zoo.disentangle import adjust_rank
    from oracle.disentangle_oracle import rank_adjust as oracle
    R = start(m)
    ar = adjust_rank()
    for k, x in enumerate(inputs(m)):
        for lvl in LVLS:
            f = ar.factors(lvl)
            ref64, S64 = oracle(x, R, f, lvl < 0.5, dtype=torch.float64)
            ref32, _ = oracle(x, R, f.astype(np.float32), lvl < 0.5, dtype=torch.float32)
            s = torch.empty(1, 20, device=DEV)
            out = ar(x.to(DEV), lvl, R=R, s_out=s).double().cpu()
            e_ref = (ref32.double() - ref64).abs().max().item()
            e_out = (out - ref64).abs().max().item()
            tol = 4 * e_ref + 1e-6 * x.std().item()
            print(f"m {m} input {k} lvl {lvl}: product {e_out:.3g}, reference fp32 {e_ref:.3g}, bound {tol:.3g}")
            assert e_out <= tol, (m, k, lvl, e_out, e_ref)
            rel = ((s.double().cpu() - S64).abs() / S64).max().item()
            assert rel <= 1e-5, (m, k, lvl, rel)


def test_batch_equals_single_calls_and_identity():
    from lib.model_zoo.disentangle import adjust_rank
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(3, 256, 768, generator=g) * torch.tensor([1.0, 0.2, 3.0])[:, None, None]).to(DEV)
    R = start(256).to(DEV)
    ar = adjust_rank()
    for lvl in (0.1, 0.9):
        batch = ar(x, lvl, R=R)
        for i in range(3):
            assert torch.equal(batch[i:i + 1], ar(x[i:i + 1], lvl, R=R)), (lvl, i)
    assert ar(x, 0.5) is x


def test_fp16_is_the_fp32_path_cast():
    from lib.model_zoo.disentangle import adjust_rank
    x = inputs(257)[0].half().to(DEV)
    R = start(257).to(DEV)
    out = adjust_rank()(x, 0.25, R=R)
    assert out.dtype == torch.float16
    assert torch.equal(out, adjust_rank()(x.float(), 0.25, R=R).half())


def test_default_start_follows_the_reference_generator():
    """Seeded: the kernel's start is torch.randn(m, 20) on the device, and the generator ends where torch.pca_lowrank leaves it."""
    from lib.model_zoo.disentangle import adjust_rank
    from oracle.disentangle_oracle import rank_adjust as oracle
    x = inputs(256)[1].to(DEV)
    torch.cuda.manual_seed(11)
    out = adjust_rank()(x, 0.75)
    state = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(11)
    R = torch.randn(256, 20, device=DEV)
    ref, _ = oracle(x.cpu(), R.cpu(), adjust_rank().factors(0.75), False, dtype=torch.float64)
    assert (out.double().cpu() - ref).abs().max().item() <= 1e-4 * x.std().item()
    torch.cuda.manual_seed(11)
    xc = x - x.mean(-1, keepdim=True)
    torch.pca_lowrank(xc, q=20, center=False, niter=1)
    assert torch.equal(torch.cuda.get_rng_state(), state)


def test_graph_capture_replays_eager_with_one_launch():
    from vdb200 import ops
    x = inputs(256)[0].to(DEV)
    R = start(256).to(DEV)
    f = torch.tensor(np.linspace(1.0, 0.0, 20), dtype=torch.float32, device=DEV)
    ops.reset_launch_count()
    eager = ops.rank_adjust(x, f, True, R)
    assert ops.launch_count() == 1
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.rank_adjust(x, f, True, R, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.rank_adjust(x, f, True, R, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_decompose_matches_oracle_factors():
    """decompose returns app.py's (u, s, v, x_mean, x_remain); u and v up to column signs."""
    from lib.model_zoo.disentangle import decompose
    from oracle.disentangle_oracle import lowrank
    x = inputs(256)[1]
    R = start(256)
    u, s, v, x_mean, x_remain = decompose(x.to(DEV), R=R.to(DEV))
    xc = (x - x.mean(-1, keepdim=True)).double()
    U, S, V = lowrank(xc, R.double(), 100)
    np.testing.assert_allclose(s.cpu().double(), S, rtol=1e-5)
    sign = torch.sign((u.cpu().double() * U).sum(1, keepdim=True))
    assert (u.cpu().double() - U * sign).abs().max().item() <= 1e-4
    assert (v.cpu().double() - V * sign).abs().max().item() <= 1e-4
    low = torch.bmm(U * S[:, None, :], V.transpose(1, 2))
    assert (x_remain.cpu().double() - (xc - low)).abs().max().item() <= 1e-4 * x.std().item()
    assert torch.allclose(x_mean.cpu(), x.mean(-1, keepdim=True), atol=1e-6)


def test_image_context_end_to_end():
    """dcg tab: CLIP image tokens, token 0 split off, locals adjusted, fed to sample_multicontext."""
    from lib.model_zoo.clip import CLIPImageContextEncoder
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.disentangle import adjust_rank
    from oracle.disentangle_oracle import rank_adjust as oracle
    from test_parity_gpu import build_net
    enc = CLIPImageContextEncoder()
    enc.allow_random_init = True
    enc.to(DEV)
    img = torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        c = enc.encode(img)
    R = start(256)
    c_loc = adjust_rank()(c[:, 1:], 0.25, R=R)
    ref, _ = oracle(c[:, 1:].cpu(), R, adjust_rank().factors(0.25), True, dtype=torch.float64)
    ref32, _ = oracle(c[:, 1:].cpu(), R, adjust_rank().factors(0.25).astype(np.float32), True, dtype=torch.float32)
    e_ref = (ref32.double() - ref).abs().max().item()
    assert (c_loc.double().cpu() - ref).abs().max().item() <= 4 * e_ref + 1e-6 * c[:, 1:].std().item()
    ci = torch.cat([c[:, :1], c_loc], dim=1)
    net, _ = build_net(mini=True)
    with torch.no_grad():
        x, _ = DDIMSampler(net).sample_multicontext(
            steps=2, shape=[1, 4, 16, 16], x_info={"type": "image", "xt": torch.randn(1, 4, 16, 16, device=DEV)},
            c_info_list=[{"type": "image", "conditioning": ci, "unconditional_conditioning": torch.zeros_like(ci),
                          "unconditional_guidance_scale": 7.5, "ratio": 1.0}], verbose=False, eta=0.)
    assert x.shape == (1, 4, 16, 16) and torch.isfinite(x).all()
