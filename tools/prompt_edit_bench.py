"""Prompt-to-Prompt editing against the unedited batch at bench.py's headline workload (BASELINE config 2): full-size synthetic
weights, 512x512 (latent 64x64), CFG 7.5, a 77-token text context, VAE decode included, every sampler on its captured step graph.
The batch is one source prompt and three targets (n = 4, bench.py's batch size).

Cases, for DDIM 50 steps and DPM-Solver++ 2M 20 steps: the unedited batch, replace, refine, and replace with a local blend
(lib/model_zoo/prompt_edit.py; cross_steps 0.8, self_steps 0.4, synthetic tables: a one-to-two token swap, an inserted word,
two blend words).  They are timed alternately, one batch (sample + decode) per sample from CUDA events, --rounds rounds (at least
3), best of; reported as ms per batch and the launches of one step, with the card name and power limit read in the same run.
graph_equals_eager: each case's graph-replayed latent equals its eager run (use_cuda_graph=False) bit for bit.
    python tools/prompt_edit_bench.py [--rounds N]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench import BS, LAT, SCALE, SEED, build_net  # noqa: E402
from lib.model_zoo.ddim import DDIMSampler  # noqa: E402
from lib.model_zoo.dpm_solver import DPMSolverSampler  # noqa: E402
from lib.model_zoo.prompt_edit import PromptEdit  # noqa: E402
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
n, L = BS, 77
c = (torch.randn(n, L, 768, generator=g) * 0.5).to(dev)
u = (torch.randn(1, L, 768, generator=g) * 0.5).repeat(n, 1, 1).to(dev)
xT = parallel.seeded_latents((0, 1), (4, LAT, LAT), seed=SEED).to(dev)

# synthetic tables: replace swaps the word at position 5 for a two-token word (weights 1/2), later positions shifted by one;
# refine inserts a token at position 3; the blend words are positions 5..6 of every row
M = np.zeros((L, L))
M[np.arange(5), np.arange(5)] = 1.0
M[5, 5] = M[5, 6] = 0.5
M[np.arange(6, L - 1), np.arange(7, L)] = 1.0
mp, alpha = np.arange(L), np.ones(L)
mp[4:] = np.arange(3, L - 1)
mp[3], alpha[3] = 3, 0.0
A_rf = np.zeros((L, L))
A_rf[mp, np.arange(L)] = alpha
w = np.zeros((n, L), np.float32)
w[:, 5:7] = 1.0
edits = {"plain": None,
         "replace": PromptEdit(np.stack([M] * (n - 1)), np.zeros((n - 1, L))),
         "refine": PromptEdit(np.stack([A_rf] * (n - 1)), np.stack([1.0 - alpha] * (n - 1))),
         "replace_blend": PromptEdit(np.stack([M] * (n - 1)), np.zeros((n - 1, L)), blend=w)}

# context buffers shared where their shapes agree: the cross-attention layers keep few K / V^T projections, and alternating
# samplers replay their captured graphs instead of re-capturing them each time
shared = {}
bufs = {"plain": shared, "replace": shared, "replace_blend": shared, "refine": {}}


def make(cls, edit, **kw):
    s = cls(net, **kw)
    s._ctx_bufs = bufs[edit]
    return s


cases = [(f"{sn}_{e}", cls, kw, steps, e) for sn, cls, kw, steps in (("ddim_50", DDIMSampler, {}, 50),
                                                                      ("dpmpp_2m_20", DPMSolverSampler, {"order": 2}, 20))
         for e in edits]
samplers = {name: make(cls, e, **kw) for name, cls, kw, _, e in cases}


def sample(smp, steps, edit):
    ci = {"type": "text", "conditioning": c, "unconditional_conditioning": u, "unconditional_guidance_scale": SCALE}
    if edits[edit] is not None:
        ci["prompt_edit"] = edits[edit]
    x_info = {"type": "image", "xt": xT.expand(n, 4, LAT, LAT).clone()}
    return smp.sample(steps=steps, shape=[n, 4, LAT, LAT], x_info=x_info, c_info=ci, verbose=False, eta=0.)[0]


res = {name: {"ms": []} for name, *_ in cases}
with torch.no_grad():
    for name, _, _, steps, e in cases:                   # warm-up: packs weights, captures each sampler's step graph
        for _ in range(2):
            net.vae_decode(sample(samplers[name], steps, e), "image")
        res[name]["launches_per_step"] = samplers[name].last_step_launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, _, _, steps, e in cases:
            torch.cuda.synchronize()
            e0.record()
            x = sample(samplers[name], steps, e)
            net.vae_decode(x, "image")
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1))
            res[name]["x"] = x
    for name, cls, kw, steps, e in cases:
        eager = sample(make(cls, e, use_cuda_graph=False, **kw), steps, e)
        r = res[name]
        x = r.pop("x")
        r["graph_equals_eager"] = bool(torch.equal(x, eager))
        r["finite"] = bool(torch.isfinite(x).all())

for name, _, _, steps, e in cases:
    r = res[name]
    ms = min(r["ms"])
    print(json.dumps(dict(card=card, case=name, steps=steps, n=n, resolution=8 * LAT, ms_per_batch=round(ms, 2),
                          ms_per_batch_all=[round(v, 2) for v in r["ms"]], launches_per_step=r["launches_per_step"],
                          graph_equals_eager=r["graph_equals_eager"], finite=r["finite"])), flush=True)
