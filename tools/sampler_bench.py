"""DDIM against multistep DPM-Solver++ at bench.py's headline workload (BASELINE config 2): full-size synthetic weights, bs 4,
512x512 (latent 64x64), CFG 7.5, a 77-token text context, VAE decode included, every sampler on its captured step graph.

Samplers: DDIM 50 steps, DPM-Solver++ 2M at 15 / 20 / 25 steps and 3M at 20 steps.  They are timed alternately, one batch
(sample + decode) per sample from CUDA events, --rounds rounds (at least 3), best of; reported as ms per batch, images/s and the
launches of one step, with the card name and power limit read in the same run.

Checks printed with the numbers:
  - graph_equals_eager: each sampler's graph-replayed latent equals its eager run (use_cuda_graph=False) bit for bit;
  - rel_l2_vs_ddim500: the relative L2 distance of each final latent to a 500-step DDIM solve from the same x_T;
  - rel_l2_vs_ddim500_same_start: the same against DDIM on the 500-point grid started at the sampler's own first grid point.
    DDIM's uniform grid, range(0, 1000, 1000 // steps) + 1, starts the walk at a different t for each step count (981 at 50
    steps, 951 at 20, 991 at 15, 999 at 500), and the same x_T read at another t starts another trajectory: the first number
    mixes that difference in, the second leaves only the discretisation error.  Both are proxies for the solver's error on the
    synthetic network: they say nothing about image quality.
    python tools/sampler_bench.py [--rounds N]"""
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
from lib.model_zoo.diffusion_utils import make_ddim_timesteps  # noqa: E402
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

# one context buffer for every sampler: the cross-attention layers then keep one set of K / V^T projections, and alternating
# samplers replay their captured graphs instead of re-capturing them each time
ctx_bufs = {}


def make(cls, **kw):
    s = cls(net, **kw)
    s._ctx_bufs = ctx_bufs
    return s


class DDIMFrom(DDIMSampler):
    """DDIM walking only the grid points at or below t_start, from the x_T it is given"""

    def __init__(self, model, t_start, **kw):
        super().__init__(model, **kw)
        self.t_start = t_start

    def _initial_latent(self, shape, x_info, dtype, device):
        x, ts = super()._initial_latent(shape, x_info, dtype, device)
        return x, ts[ts <= self.t_start]


samplers = {"ddim": make(DDIMSampler), "dpmpp_2m": make(DPMSolverSampler, order=2), "dpmpp_3m": make(DPMSolverSampler, order=3)}
cases = [("ddim_50", "ddim", 50), ("dpmpp_2m_15", "dpmpp_2m", 15), ("dpmpp_2m_20", "dpmpp_2m", 20),
         ("dpmpp_2m_25", "dpmpp_2m", 25), ("dpmpp_3m_20", "dpmpp_3m", 20)]


def sample(smp, steps):
    return smp.sample(steps=steps, shape=[BS, 4, LAT, LAT], x_info={"type": "image", "xt": xT.clone()},
                      c_info={"type": "text", "conditioning": c, "unconditional_conditioning": u,
                              "unconditional_guidance_scale": SCALE}, verbose=False, eta=0.)[0]


res = {name: {"ms": []} for name, _, _ in cases}
with torch.no_grad():
    for name, key, steps in cases:                    # warm-up: packs weights, captures each sampler's step graph
        for _ in range(2):
            net.vae_decode(sample(samplers[key], steps), "image")
        res[name]["launches_per_step"] = samplers[key].last_step_launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, key, steps in cases:
            torch.cuda.synchronize()
            e0.record()
            x = sample(samplers[key], steps)
            net.vae_decode(x, "image")
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1))
            res[name]["x"] = x
    ref = sample(make(DDIMSampler), 500).double()
    same_start = {}
    for name, key, steps in cases:
        t_start = int(make_ddim_timesteps("uniform", steps, 1000, verbose=False)[-1])
        if t_start not in same_start:
            same_start[t_start] = sample(make(DDIMFrom, t_start=t_start), 500).double()
        res[name]["t_start"] = t_start
    for name, key, steps in cases:
        cls, kw = (DDIMSampler, {}) if key == "ddim" else (DPMSolverSampler, {"order": samplers[key].order})
        eager = sample(make(cls, use_cuda_graph=False, **kw), steps)
        r = res[name]
        r["graph_equals_eager"] = bool(torch.equal(r.pop("x"), eager))
        r["rel_l2_vs_ddim500"] = float((eager.double() - ref).norm() / ref.norm())
        ref_s = same_start[r["t_start"]]
        r["rel_l2_vs_ddim500_same_start"] = float((eager.double() - ref_s).norm() / ref_s.norm())
        r["finite"] = bool(torch.isfinite(eager).all())

for name, key, steps in cases:
    r = res[name]
    ms = min(r["ms"])
    print(json.dumps(dict(card=card, sampler=name, steps=steps, bs=BS, resolution=8 * LAT, ms_per_batch=round(ms, 2),
                          ms_per_batch_all=[round(v, 2) for v in r["ms"]], images_per_s=round(BS * 1e3 / ms, 3),
                          launches_per_step=r["launches_per_step"], graph_equals_eager=r["graph_equals_eager"], finite=r["finite"],
                          t_start=r["t_start"], rel_l2_vs_ddim500=round(r["rel_l2_vs_ddim500"], 5),
                          rel_l2_vs_ddim500_same_start=round(r["rel_l2_vs_ddim500_same_start"], 5))), flush=True)
