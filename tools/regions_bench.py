"""Region prompts (lib/model_zoo/regions.py): full-size synthetic weights, CFG 7.5, 77-token text contexts, VAE decode included.

Cases, alternated round by round, best of --rounds:
  - bench.py's config 2 (bs 4 at 512x512, DDIM 50, 8 UNet items per step), plain, the yardstick for ms per UNet item;
  - config 2's shape with R = 1, 2, 4 regions (left-to-right vertical bands), bootstrapping off and on (the first 20 % of the
    steps, white and black backgrounds), for DDIM 50 and DPM-Solver++ 2M 20, on the captured step graph; R = 2 with
    bootstrapping also eagerly (use_cuda_graph=False), to check that the graph latent equals the eager one bit for bit;
  - a 512x2048 panorama (windows of 64 at stride 16, 13 windows) with 2 regions, DDIM 50 and DPM-Solver++ 2M 20.
Per case: ms per call (sample + decode), ms per step, UNet items and launches per step, ms per UNet item.  Then:
  - chunk sweep: the panorama case under DPM-Solver++ 20 with 1, 2 and 4 windows per UNet call (the default is
    WINDOWS_PER_CHUNK // (R + 1) = 2);
  - gather + merge alone: one step's region gathers and merges at config 2's shape (R = 2, bootstrapping on) captured in a CUDA
    graph and replayed between CUDA events.
The card name and power limit are read in the same run.
    python tools/regions_bench.py [--rounds N]"""
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
from lib.model_zoo import panorama  # noqa: E402
from lib.model_zoo.ddim import DDIMSampler  # noqa: E402
from lib.model_zoo.dpm_solver import DPMSolverSampler  # noqa: E402
from lib.model_zoo.regions import Region, Regions  # noqa: E402
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
c1 = (torch.randn(1, 77, 768, generator=g) * 0.5).to(dev)
u1 = (torch.randn(1, 77, 768, generator=g) * 0.5).to(dev)
rc = [(torch.randn(1, 77, 768, generator=g) * 0.5).to(dev) for _ in range(4)]
BGS = torch.tensor([[0.9, 0.1, -0.2, 0.3], [-0.6, 0.4, 0.2, -0.1]], device=dev)
PH, PW = 64, 256
xT2 = parallel.seeded_latents((0, BS), (4, LAT, LAT), seed=SEED).to(dev)
xTp = parallel.seeded_latents((0, 1), (4, PH, PW), seed=SEED).to(dev)
SAMPLERS = {"ddim": (DDIMSampler, {}, 50), "dpmpp_2m": (DPMSolverSampler, {"order": 2}, 20)}


def bands(R, H, W):
    """R vertical bands, each the r-th fifth-overlapping strip of the width"""
    out = []
    for r in range(R):
        m = torch.zeros(1, H, W, device=dev)
        m[..., r * W // (R + 1):(r + 2) * W // (R + 1)] = 1.0
        out.append(m)
    return out


def regions_of(R, boot_steps, n, H, W):
    return Regions([Region(m, rc[r].repeat(n, 1, 1)) for r, m in enumerate(bands(R, H, W))], bootstrap_steps=boot_steps,
                   backgrounds=BGS if boot_steps else None)


# case: (name, sampler kind, R (0: plain), bootstrap, panorama, graph)
cases = [("config2_ddim_50", "ddim", 0, False, False, True)]
for kind in SAMPLERS:
    for R in (1, 2, 4):
        for boot in (False, True):
            cases.append((f"{kind}_{SAMPLERS[kind][2]}_R{R}_{'boot' if boot else 'noboot'}", kind, R, boot, False, True))
    cases.append((f"{kind}_{SAMPLERS[kind][2]}_R2_boot_eager", kind, 2, True, False, False))
    cases.append((f"{kind}_{SAMPLERS[kind][2]}_panorama512x2048_R2", kind, 2, False, True, True))

# shared context buffers, as panorama_bench.py does, so alternating samplers replay their captured graphs
ctx_bufs = {}


def make(name, kind, graph):
    cls, kw, _ = SAMPLERS[kind]
    s = cls(net, use_cuda_graph=graph, **kw)
    s._ctx_bufs = ctx_bufs.setdefault(name.replace("_eager", ""), {})
    return s


def sample(smp, kind, R, boot, pano):
    steps = SAMPLERS[kind][2]
    n, H, W, xT = (1, PH, PW, xTp) if pano else (BS, LAT, LAT, xT2)
    x_info = {"type": "image", "xt": xT.clone()}
    if R:
        x_info["regions"] = regions_of(R, steps // 5 if boot else 0, n, H, W)
    if pano:
        x_info["windows"] = panorama.Windows(64, 16)
    torch.manual_seed(0)
    return smp.sample(steps=steps, shape=[n, 4, H, W], x_info=x_info, c_info={"type": "text", "conditioning": c1.repeat(n, 1, 1),
                      "unconditional_conditioning": u1.repeat(n, 1, 1), "unconditional_guidance_scale": SCALE},
                      verbose=False, eta=0.)[0]


def items_per_step(R, boot, pano):
    if not R:
        return 2 * BS
    nwin = panorama.layout(panorama.Windows(64, 16), PH, PW).nwin if pano else 1
    return nwin * (1 if pano else BS) * ((R + 1 if boot else 1) + R + 1)


samplers = {name: make(name, kind, graph) for name, kind, _, _, _, graph in cases}
e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def timed(name, kind, R, boot, pano):
    torch.cuda.synchronize()
    e[0].record()
    x = sample(samplers[name], kind, R, boot, pano)
    e[1].record()
    net.vae_decode(x, "image")
    e[2].record()
    torch.cuda.synchronize()
    return x, e[0].elapsed_time(e[1]), e[0].elapsed_time(e[2])


res = {name: {"call": [], "sample": []} for name, *_ in cases}
with torch.no_grad():
    for name, kind, R, boot, pano, _ in cases:       # warm-up: packs weights, captures each graph sampler's step graph
        timed(name, kind, R, boot, pano)
        res[name]["launches_per_step"] = getattr(samplers[name], "last_step_launches", None)
    for _ in range(args.rounds):
        for name, kind, R, boot, pano, _ in cases:
            x, ms_sample, ms_call = timed(name, kind, R, boot, pano)
            res[name]["call"].append(ms_call)
            res[name]["sample"].append(ms_sample)
            res[name]["x"] = x

c2_item = min(res["config2_ddim_50"]["sample"]) / 50 / (2 * BS)
for name, kind, R, boot, pano, graph in cases:
    r = res[name]
    steps = SAMPLERS[kind][2]
    items = items_per_step(R, boot, pano)
    out = dict(card=card, case=name, steps=steps, regions=R, bootstrap_steps=steps // 5 if boot else 0,
               resolution="512x2048 stride 16" if pano else "512x512 bs 4", graph=graph,
               ms_per_call=round(min(r["call"]), 2), ms_per_call_all=[round(v, 1) for v in r["call"]],
               ms_per_step=round(min(r["sample"]) / steps, 3), unet_items_per_step=items,
               launches_per_step=r["launches_per_step"], ms_per_unet_item=round(min(r["sample"]) / steps / items, 4),
               config2_ms_per_unet_item=round(c2_item, 4), finite=bool(torch.isfinite(r["x"]).all()))
    if not graph:
        out["graph_equals_eager"] = bool(torch.equal(r["x"], res[name.replace("_eager", "")]["x"]))
    print(json.dumps(out), flush=True)

# ---- chunk sweep -----------------------------------------------------------------------------------------------------------------
for name in list(samplers):
    del samplers[name]
res = None
torch.cuda.synchronize()
torch.cuda.empty_cache()
default_chunk = panorama.WINDOWS_PER_CHUNK
with torch.no_grad():
    for per in (1, 2, 4):
        panorama.WINDOWS_PER_CHUNK = per * 3           # R = 2: WINDOWS_PER_CHUNK // (R + 1) windows per UNet call
        s = make(f"sweep{per}", "dpmpp_2m", True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        sample(s, "dpmpp_2m", 2, False, True)
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ms = []
        for _ in range(3):
            e[0].record()
            sample(s, "dpmpp_2m", 2, False, True)
            e[1].record()
            torch.cuda.synchronize()
            ms.append(e[0].elapsed_time(e[1]))
        print(json.dumps(dict(card=card, case="chunk_sweep_dpmpp_2m_20_panorama_R2", windows_per_call=per,
                              ms_per_step=round(min(ms) / 20, 3), sample_peak_mb_above_allocated=round(peak, 1),
                              launches_per_step=s.last_step_launches)), flush=True)
        del s
    panorama.WINDOWS_PER_CHUNK = default_chunk

    # ---- gather + merge alone at config 2's shape, R = 2, bootstrapping on --------------------------------------------------------
    s = make("gm", "ddim", True)
    sample(s, "ddim", 2, True, False)
    st = s._st
    rs = st["regions"]
    mode_ub, R = 3, 2
    eps_in = torch.randn_like(rs.xw)

    def gm():
        ops.region_gather(st["x_in"][:BS], rs.oy, rs.ox, LAT, LAT, 0, 1, R, mode_ub, out=rs.xw, masks=rs.masks, rows=rs.rows,
                          step_idx=st["idx"], seed=rs.seed, bg=rs.bg)
        ops.region_merge(eps_in, rs.oy, rs.ox, rs.cover_y, rs.cover_x, 0, 1, R, rs.masks, rs.eps, halves=2)

    st["idx"].fill_(49)                                # a bootstrapped step: the gather draws its noise
    gm()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        gm()
    for _ in range(10):
        gr.replay()
    reps = 200
    e[0].record()
    for _ in range(reps):
        gr.replay()
    e[1].record()
    torch.cuda.synchronize()
    print(json.dumps(dict(card=card, case="gather_merge_per_step_config2_R2_boot", ms_per_step=round(e[0].elapsed_time(e[1]) / reps, 4),
                          launches=2)), flush=True)
