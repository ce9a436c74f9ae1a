"""Self-attention guidance against unguided sampling at bench.py's headline workload (BASELINE config 2): full-size synthetic
weights, bs 4, 512x512 (latent 64x64), CFG 7.5, a 77-token text context, VAE decode included, every sampler on its captured step
graph.

Cases: DDIM 50 steps and DPM-Solver++ 2M 20 steps, each without SAG and with SAG at scale 0.75 (lib/model_zoo/sag.py), from the
same x_T.  They are timed alternately from CUDA events, --rounds rounds (at least 3), best of: ms per batch (sample + decode) and
ms per step (the sample alone over its steps), with the UNet items and the launches of one step, and the card name and power limit
read in the same run.  graph_equals_eager: each case's graph-replayed latent equals its eager run (use_cuda_graph=False) bit for
bit; eager_ms_per_batch times that eager run.  sag_kernels: the three SAG entry points of one step at this shape (the mid block's
key mass of bs uncond rows, N = 8 x 8 tokens, 8 heads, d_head 160, on the fused q | k layout; the degrade; the guide) captured
alone in a CUDA graph and replayed 200 times: us per step and their share of a SAG step.
    python tools/sag_bench.py [--rounds N]"""
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
from lib.model_zoo.sag import SelfAttentionGuidance, mid_size  # noqa: E402
from vdb200 import ops, parallel  # noqa: E402

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

# one context buffer for every sampler: the cross-attention layers keep one set of K / V^T projections, and alternating
# samplers replay their captured graphs instead of re-capturing them each time
ctx_bufs = {}


def make(cls, **kw):
    s = cls(net, **kw)
    s._ctx_bufs = ctx_bufs
    return s


cases = [("ddim_50", DDIMSampler, {}, 50, False), ("ddim_50_sag", DDIMSampler, {}, 50, True),
         ("dpmpp_2m_20", DPMSolverSampler, {"order": 2}, 20, False), ("dpmpp_2m_20_sag", DPMSolverSampler, {"order": 2}, 20, True)]
samplers = {name: make(cls, **kw) for name, cls, kw, _, _ in cases}


def sample(smp, steps, sag):
    x_info = {"type": "image", "xt": xT.clone()}
    if sag:
        x_info["sag"] = SelfAttentionGuidance(0.75)
    torch.manual_seed(0)
    return smp.sample(steps=steps, shape=[BS, 4, LAT, LAT], x_info=x_info,
                      c_info={"type": "text", "conditioning": c, "unconditional_conditioning": u,
                              "unconditional_guidance_scale": SCALE}, verbose=False, eta=0.)[0]


def sag_kernels_us():
    """the three SAG entry points of one step at this shape, alone in a captured graph -> us per step"""
    H, d = 8, 160
    dk = ops.attention_pads(d)[0]
    hm, wm = mid_size(LAT, LAT)
    N = hm * wm
    gk = torch.Generator(device=dev).manual_seed(3)
    qk = (torch.randn(2 * BS * N, 2 * H * dk, generator=gk, device=dev) * 0.5).to(torch.bfloat16)
    mass = torch.zeros(BS, N, device=dev)
    x, e = (torch.randn(BS, LAT, LAT, 4, generator=gk, device=dev) for _ in range(2))
    eps = torch.randn(2 * BS, LAT, LAT, 4, generator=gk, device=dev)
    table = torch.tensor([[0.8, 0.6]], device=dev)
    idx = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.empty_like(x)

    def step():
        mass.zero_()
        ops.sattn_key_mass(qk, qk, mass, 0, H, N, d, w=1.0 / H, q_col0=0, k_col0=H * dk)
        ops.sag_degrade(x, e, mass, table, idx, hm, wm, out=out)
        ops.sag_guide(eps[:BS], eps[BS:], out, 0.75)

    step()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = None
    for _ in range(5):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(200):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / 200
        best = us if best is None else min(best, us)
    return best


res = {name: {"ms": [], "ms_sample": []} for name, _, _, _, _ in cases}
with torch.no_grad():
    for name, _, _, steps, sag in cases:              # warm-up: packs weights, captures each sampler's step graph
        for _ in range(2):
            net.vae_decode(sample(samplers[name], steps, sag), "image")
        res[name]["launches_per_step"] = samplers[name].last_step_launches
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    for _ in range(args.rounds):
        for name, _, _, steps, sag in cases:
            torch.cuda.synchronize()
            e0.record()
            x = sample(samplers[name], steps, sag)
            e1.record()
            net.vae_decode(x, "image")
            e2.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e2))
            res[name]["ms_sample"].append(e0.elapsed_time(e1))
            res[name]["x"] = x
    for name, cls, kw, steps, sag in cases:
        torch.cuda.synchronize()
        e0.record()
        eager = sample(make(cls, use_cuda_graph=False, **kw), steps, sag)
        net.vae_decode(eager, "image")
        e2.record()
        torch.cuda.synchronize()
        r = res[name]
        r["eager_ms"] = e0.elapsed_time(e2)
        x = r.pop("x")
        r["graph_equals_eager"] = bool(torch.equal(x, eager))
        r["finite"] = bool(torch.isfinite(x).all())
    kern_us = sag_kernels_us()

for name, _, _, steps, sag in cases:
    r = res[name]
    ms, ms_step = min(r["ms"]), min(r["ms_sample"]) / steps
    out = dict(card=card, case=name, steps=steps, bs=BS, resolution=8 * LAT, ms_per_batch=round(ms, 2),
               ms_per_batch_all=[round(v, 2) for v in r["ms"]], ms_per_step=round(ms_step, 3),
               unet_items_per_step=(3 if sag else 2) * BS, launches_per_step=r["launches_per_step"],
               eager_ms_per_batch=round(r["eager_ms"], 2), graph_equals_eager=r["graph_equals_eager"], finite=r["finite"])
    if sag:
        out["sag_kernels_us_per_step"] = round(kern_us, 2)
        out["sag_kernels_share_of_step"] = round(kern_us * 1e-3 / ms_step, 5)
    print(json.dumps(out), flush=True)
