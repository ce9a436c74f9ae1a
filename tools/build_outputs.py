"""Bit-for-bit comparison of two builds on the seeded workloads bench.py does not run.

A change that must not alter any arithmetic (a refactor of the kernel layer) has to compute exactly what its parent computed.
bench.py --dump-outputs covers the benchmark's own configs; this script covers the other paths, on the mini models of the
parity tests (synthetic seeded weights):
  * DPM-Solver++ 2M-20 (CFG 7.5, 32x32 latent, bs 2),
  * an inpainting DDIM walk (soft latent mask, Philox noise keyed by torch.manual_seed),
  * the text-latent diffuser (4-step DDIM on a [2, 768] latent, image context),
  * a VAE decode whose Upsamples all take the folded path (64x64 latent) and one whose Upsamples all take the unfolded path
    (8x8 latent),
  * a CLIP text encode and a CLIP image encode (quick_gelu MLPs) and a 2-layer Optimus BERT encode (GELU feed-forward), on
    synthetic seeded weights as in the CLIP and text-encoder tests.

Each build runs with its own tree's Python and library; then the dumps are compared with torch.equal:

    python <tree A>/tools/build_outputs.py --dump a.pt
    python <tree B>/tools/build_outputs.py --dump b.pt
    python tools/build_outputs.py --compare a.pt b.pt
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))

import torch  # noqa: E402

DEV = "cuda"


def build_net(text_flows=False):
    """the mini VD net of the parity tests: model_channels 64, VAE ch 64, seeded synthetic weights"""
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
    from oracle import weights
    from oracle.make_golden import MINI_UNET, MINI_VAE, WEIGHT_SEED
    cfg = model_cfg_bank()('vd_four_flow_v1-0')
    if text_flows:
        cfg.args.diffuser_cfg_list[1][1] = model_cfg_bank()('openai_unet_0d_v1_dc')
        cfg.args.vae_cfg_list = []
    cfg.args.ctx_cfg_list = []
    for _, d in cfg.args.diffuser_cfg_list:
        d.args.update(MINI_UNET)
    if not text_flows:
        cfg.args.vae_cfg_list[0][1].args.ddconfig.update(MINI_VAE)
    net = get_model()(cfg, verbose=False)
    net.load_state_dict(weights.synth_state_dict(weights.param_shapes(net), seed=WEIGHT_SEED), strict=False)
    net.eval()
    net.to(DEV)
    return net


def cinfo(c, u, typ="text"):
    return {"type": typ, "conditioning": c.to(DEV), "unconditional_conditioning": u.to(DEV), "unconditional_guidance_scale": 7.5}


def synth_encoder(cfg_name, seed=3):
    """a CLIP context encoder of the config bank with seeded synthetic weights"""
    from lib.cfg_helper import model_cfg_bank
    from lib.model_zoo import get_model
    from oracle import weights
    enc = get_model()(model_cfg_bank()(cfg_name), verbose=False)
    shapes = {k: tuple(v.shape) for k, v in enc.model.named_parameters()}
    enc.model.load_state_dict(weights.synth_state_dict(shapes, seed=seed), strict=False)
    return enc.to(DEV)


def synth_bert(n_layer=2, seed=7):
    """the Optimus BERT encoder with seeded synthetic weights"""
    from lib.model_zoo.optimus import optimus_vae_next
    from oracle import weights
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=1)), encoder=dict(config=dict(num_hidden_layers=n_layer)))
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("encoder.")}
    m.load_state_dict({k: weights.tensor_for(k, s, seed) for k, s in shapes.items()}, strict=False)
    return m.to(DEV)


def run_encoders(g):
    out = {}
    with torch.no_grad():
        tok = torch.full((3, 77), 49407, dtype=torch.long)
        tok[:, 0] = 49406
        for i in range(3):
            tok[i, 1:6 + 7 * i] = torch.randint(1000, 40000, (5 + 7 * i,), generator=g)
        enc = synth_encoder("clip_text_context_encoder")
        out["clip_text_encode"] = enc.encode_tokens(tok)
        del enc
        enc = synth_encoder("clip_image_context_encoder")
        out["clip_image_encode"] = enc.encode(torch.rand(2, 3, 300, 360, generator=g).to(DEV))
        del enc
        lengths = [9, 70, 33, 79]
        ids = torch.zeros(len(lengths), max(lengths), dtype=torch.long)
        for r, n in enumerate(lengths):
            ids[r, 0], ids[r, n - 1] = 101, 102
            ids[r, 1:n - 1] = torch.randint(999, 28996, (n - 2,), generator=g)
        out["bert_encode"] = synth_bert().encode_ids(ids, lengths)
    return out


def run_cases():
    from lib.model_zoo.ddim import DDIMSampler
    from lib.model_zoo.dpm_solver import DPMSolverSampler
    out = {}
    g = torch.Generator().manual_seed(1234)
    net = build_net()
    with torch.no_grad():
        c, u = torch.randn(2, 77, 768, generator=g) * 0.5, torch.randn(2, 77, 768, generator=g) * 0.5
        xT = torch.randn(2, 4, 32, 32, generator=g)
        out["dpmpp_2m_20"] = DPMSolverSampler(net, order=2).sample(
            steps=20, shape=[2, 4, 32, 32], x_info={"type": "image", "xt": xT.to(DEV)}, c_info=cinfo(c, u),
            verbose=False, eta=0.)[0]

        x0 = torch.randn(2, 4, 32, 32, generator=g) * 0.8
        mask = torch.zeros(2, 1, 32, 32)
        mask[:, :, :, 14:] = 1.0
        mask[:, :, :, 12:14] = 0.5
        torch.manual_seed(7)
        out["inpaint_ddim_10"] = DDIMSampler(net).sample(
            steps=10, shape=[2, 4, 32, 32],
            x_info={"type": "image", "xt": xT.to(DEV), "x0": x0.to(DEV), "inpaint_mask": mask.to(DEV)},
            c_info=cinfo(c, u), verbose=False, eta=0.)[0]

        out["vae_decode_folded_64"] = net.vae_decode(torch.randn(1, 4, 64, 64, generator=g).to(DEV), "image")
        out["vae_decode_unfolded_8"] = net.vae_decode(torch.randn(2, 4, 8, 8, generator=g).to(DEV), "image")
    del net
    net = build_net(text_flows=True)
    with torch.no_grad():
        xt = torch.randn(2, 768, generator=g)
        ci, ui = torch.randn(2, 257, 768, generator=g) * 0.5, torch.zeros(2, 257, 768)
        out["text_latent_ddim_4"] = DDIMSampler(net).sample(
            steps=4, shape=[2, 768], x_info={"type": "text", "xt": xt.to(DEV)}, c_info=cinfo(ci, ui, "image"),
            verbose=False, eta=0.)[0]
    del net
    out.update(run_encoders(g))
    return {k: v.detach().cpu() for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dump", metavar="FILE")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.dump:
        res = run_cases()
        torch.save(res, args.dump)
        for k, v in res.items():
            print(f"{k}: {tuple(v.shape)} {v.dtype} finite {bool(torch.isfinite(v.float()).all())}")
    if args.compare:
        a, b = (torch.load(p) for p in args.compare)
        ok = set(a) == set(b)
        for k in sorted(set(a) | set(b)):
            same = k in a and k in b and a[k].dtype == b[k].dtype and torch.equal(a[k], b[k])
            ok &= same
            print(f"{k}: {'identical' if same else 'DIFFERENT'}")
        print("all identical" if ok else "builds differ")
        sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
