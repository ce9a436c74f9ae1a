"""Inpainting against plain sampling at bench.py's headline workload (BASELINE config 2): full-size synthetic weights, bs 4,
512x512 (latent 64x64), CFG 7.5, a 77-token text context, VAE decode included, every sampler on its captured step graph.

Cases: DDIM 50 steps and DPM-Solver++ 2M 20 steps, each without a mask and with a soft per-item latent mask (the blend of
lib/model_zoo/inpaint.py after every step, full walk from the same x_T).  They are timed alternately, one batch (sample +
decode) per sample from CUDA events, --rounds rounds (at least 3), best of; reported as ms per batch and the launches of one
step, with the card name and power limit read in the same run.  graph_equals_eager: each case's graph-replayed latent equals
its eager run (use_cuda_graph=False) bit for bit under the same torch seed.
    python tools/inpaint_bench.py [--rounds N]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))
import torch  # noqa: E402
from bench import BS, LAT, SCALE, SEED, build_net  # noqa: E402
from lib.model_zoo.ddim import DDIMSampler  # noqa: E402
from lib.model_zoo.dpm_solver import DPMSolverSampler  # noqa: E402
from vdb200 import parallel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
if args.rounds < 3:
    raise SystemExit("--rounds must be at least 3")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card, flush=True)
net = build_net(dev)
g = torch.Generator().manual_seed(2)
c = (torch.randn(1, 77, 768, generator=g) * 0.5).repeat(BS, 1, 1).to(dev)
u = (torch.randn(1, 77, 768, generator=g) * 0.5).repeat(BS, 1, 1).to(dev)
xT = parallel.seeded_latents((0, BS), (4, LAT, LAT), seed=SEED).to(dev)
x0 = (torch.randn(BS, 4, LAT, LAT, generator=g) * 0.8).to(dev)
mask = torch.zeros(BS, 1, LAT, LAT)
for b in range(BS):                                  # regenerate a square per item, with a soft one-cell border
    lo, hi = 8 + 4 * b, 40 + 4 * b
    mask[b, :, lo - 1:hi + 1, lo - 1:hi + 1] = 0.5
    mask[b, :, lo:hi, lo:hi] = 1.0
mask = mask.to(dev)

# one context buffer for every sampler: the cross-attention layers keep one set of K / V^T projections, and alternating
# samplers replay their captured graphs instead of re-capturing them each time
ctx_bufs = {}


def make(cls, **kw):
    s = cls(net, **kw)
    s._ctx_bufs = ctx_bufs
    return s


cases = [("ddim_50", DDIMSampler, {}, 50, False), ("ddim_50_inpaint", DDIMSampler, {}, 50, True),
         ("dpmpp_2m_20", DPMSolverSampler, {"order": 2}, 20, False), ("dpmpp_2m_20_inpaint", DPMSolverSampler, {"order": 2}, 20, True)]
samplers = {name: make(cls, **kw) for name, cls, kw, _, _ in cases}


def sample(smp, steps, masked):
    x_info = {"type": "image", "xt": xT.clone()}
    if masked:
        x_info.update(x0=x0, inpaint_mask=mask)
    torch.manual_seed(0)
    return smp.sample(steps=steps, shape=[BS, 4, LAT, LAT], x_info=x_info,
                      c_info={"type": "text", "conditioning": c, "unconditional_conditioning": u,
                              "unconditional_guidance_scale": SCALE}, verbose=False, eta=0.)[0]


res = {name: {"ms": []} for name, _, _, _, _ in cases}
with torch.no_grad():
    for name, _, _, steps, masked in cases:              # warm-up: packs weights, captures each sampler's step graph
        for _ in range(2):
            net.vae_decode(sample(samplers[name], steps, masked), "image")
        res[name]["launches_per_step"] = samplers[name].last_step_launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, _, _, steps, masked in cases:
            torch.cuda.synchronize()
            e0.record()
            x = sample(samplers[name], steps, masked)
            net.vae_decode(x, "image")
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1))
            res[name]["x"] = x
    for name, cls, kw, steps, masked in cases:
        eager = sample(make(cls, use_cuda_graph=False, **kw), steps, masked)
        r = res[name]
        x = r.pop("x")
        r["graph_equals_eager"] = bool(torch.equal(x, eager))
        r["finite"] = bool(torch.isfinite(x).all())
        if masked:
            keep = (mask == 0).expand_as(x)
            r["kept_region_is_x0"] = bool(torch.equal(x[keep], x0[keep]))

for name, _, _, steps, masked in cases:
    r = res[name]
    ms = min(r["ms"])
    out = dict(card=card, case=name, steps=steps, bs=BS, resolution=8 * LAT, ms_per_batch=round(ms, 2),
               ms_per_batch_all=[round(v, 2) for v in r["ms"]], images_per_s=round(BS * 1e3 / ms, 3),
               launches_per_step=r["launches_per_step"], graph_equals_eager=r["graph_equals_eager"], finite=r["finite"])
    if masked:
        out["kept_region_is_x0"] = r["kept_region_is_x0"]
    print(json.dumps(out), flush=True)
