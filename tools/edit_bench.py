"""Editing (lib/model_zoo/edit.py) at bench.py's headline workload (BASELINE config 2): full-size synthetic weights, bs 4, 512x512
(latent 64x64), 77-token text contexts, DDIM 50, CFG 7.5 for the target, VAE decode included, every walk on its captured step graph.

Per strength (0.5 and 1.0, k = int(50 * strength) grid points), each part timed alone from CUDA events, --rounds rounds, best of:
  invert   the inversion walk under the source prompt at scale 1 (k steps)
  mask     diffedit_mask with D = 10 draws (one UNet call per side, batch 40 and 80)
  regen    the masked walk from the inversion under the target prompt (k steps)
  decode   the VAE decode
  img2img  plain img2img at the same strength (x0_forward_timesteps = min(k, 49), that many steps + decode), the yardstick
Round 0 warms up (packs weights, captures each walk's step graph); in the timed rounds every walk replays its cached graph
(timed_rounds_only_replay: no eager step ran in them): the regeneration and img2img run on two samplers that share their
context buffers.  ms_per_step divides a walk's time by its
steps.  Reported with the launches of the eager step before each capture, and the card name and power limit read in the same
run.
graph_equals_eager: the inversion's trajectory and the regenerated latent of the graph path equal the eager path
(use_cuda_graph=False) bit for bit.
    python tools/edit_bench.py [--rounds N]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))
import torch  # noqa: E402
from bench import BS, LAT, SCALE, build_net  # noqa: E402
from lib.model_zoo.ddim import DDIMSampler  # noqa: E402
from lib.model_zoo.edit import diffedit_mask  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()
if args.rounds < 1:
    raise SystemExit("--rounds must be at least 1")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
net = build_net(dev)
g = torch.Generator().manual_seed(2)
u = (torch.randn(1, 77, 768, generator=g) * 0.5).repeat(BS, 1, 1).to(dev)
c_src = (torch.randn(1, 77, 768, generator=g) * 0.5).repeat(BS, 1, 1).to(dev)
c_tgt = c_src.clone()
c_tgt[:, 3:9] = (torch.randn(1, 6, 768, generator=g) * 0.5).to(dev)       # the prompt differs in a few tokens
x0 = (torch.randn(BS, 4, LAT, LAT, generator=g) * 0.8).to(dev)
STEPS, D = 50, 10
shape = [BS, 4, LAT, LAT]


def cinfo(c, s):
    return {"type": "text", "conditioning": c, "unconditional_conditioning": u, "unconditional_guidance_scale": s}


src, src1, tgt = cinfo(c_src, SCALE), cinfo(c_src, 1.0), cinfo(c_tgt, SCALE)
# a sampler keeps one sampling graph, so the masked regeneration (S) and img2img (S_i2i) run on their own samplers; they share
# the context buffers, so the cross-attention layers keep one set of K / V^T projections and both replay their cached graphs
ctx_bufs = {}
S, S_i2i = DDIMSampler(net), DDIMSampler(net)
S._ctx_bufs = S_i2i._ctx_bufs = ctx_bufs
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def timed(fn):
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def regen(smp, inv, mask):
    return smp.sample(steps=STEPS, shape=shape, x_info={"type": "image", "inversion": inv, "inpaint_mask": mask}, c_info=tgt,
                      verbose=False, eta=0.)[0]


def img2img(k):
    # the img2img start noises x0 to grid point k, so it walks at most n - 1 points: strength 1.0 runs 49 steps
    k = min(k, STEPS - 1)                               # the 'uniform' grid of 50 steps has 50 points
    return S_i2i.sample(steps=STEPS, shape=shape, x_info={"type": "image", "x0": x0, "x0_forward_timesteps": k}, c_info=tgt,
                    verbose=False, eta=0.)[0]


with torch.no_grad():
    for strength in (0.5, 1.0):
        k = int(STEPS * strength)
        parts = {p: [] for p in ("invert", "mask", "regen", "decode", "img2img")}
        launches = {}
        for r in range(args.rounds + 1):                   # round 0 warms up: packs weights, captures the step graphs
            inv, ms_inv = timed(lambda: S.invert(STEPS, x0, src1, k=k))
            torch.manual_seed(0)
            mask, ms_mask = timed(lambda: diffedit_mask(net, x0, src, tgt, steps=STEPS, strength=strength, n_draws=D))
            z, ms_regen = timed(lambda: regen(S, inv, mask))
            _, ms_dec = timed(lambda: net.vae_decode(z, "image"))
            if r == 0:
                launches = {"invert_step": S.last_invert_step_launches, "masked_step": S.last_step_launches}
            _, ms_i2i = timed(lambda: net.vae_decode(img2img(k), "image"))
            if r == 0:
                launches["img2img_step"] = S_i2i.last_step_launches
                # the eager step before a capture sets these again: they stay None while every timed walk only replays
                S.last_step_launches = S.last_invert_step_launches = S_i2i.last_step_launches = None
                continue
            for p, v in zip(parts, (ms_inv, ms_mask, ms_regen, ms_dec, ms_i2i)):
                parts[p].append(v)
        replayed = S.last_step_launches is None and S.last_invert_step_launches is None and S_i2i.last_step_launches is None
        eager = DDIMSampler(net, use_cuda_graph=False)
        inv_e = eager.invert(STEPS, x0, src1, k=k)
        z_e = regen(eager, inv_e, mask)
        keep = (mask == 0).expand_as(z)
        best = {p: round(min(v), 2) for p, v in parts.items()}
        out = dict(card=card, steps=STEPS, strength=strength, k=k, bs=BS, resolution=8 * LAT, n_draws=D,
                   ms=best, ms_all={p: [round(x, 2) for x in v] for p, v in parts.items()},
                   ms_edit_total=round(best["invert"] + best["mask"] + best["regen"] + best["decode"], 2),
                   ms_per_step={"invert": round(best["invert"] / k, 3), "regen": round(best["regen"] / k, 3),
                                "img2img_with_decode": round(best["img2img"] / min(k, STEPS - 1), 3)},
                   launches_per_step=launches, timed_rounds_only_replay=replayed, mask_fraction=round(mask.mean().item(), 4),
                   graph_equals_eager=bool(torch.equal(inv_e.trajectory, inv.trajectory) and torch.equal(z_e, z)),
                   kept_region_is_x0=bool(torch.equal(z[keep], x0[keep])), finite=bool(torch.isfinite(z).all()))
        print(json.dumps(out), flush=True)
