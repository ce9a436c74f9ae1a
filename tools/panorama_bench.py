"""Panoramas (lib/model_zoo/panorama.py) at 512x2048 (latent 64x256): full-size synthetic weights, n = 1, CFG 7.5, a 77-token
text context, VAE decode included.

Cases: DDIM 50 steps and DPM-Solver++ 2M 20 steps, each at window stride 8 (25 windows of 64x64) and 16 (13 windows), on the
captured step graph and eagerly (use_cuda_graph=False), alternated round by round; bench.py's config 2 (bs 4 at 512x512 under
CFG: 8 UNet items per step, DDIM 50) runs in the same rounds as the yardstick for ms per UNet item.  Per case, best of --rounds:
ms per call (sample + decode), ms per step (sample only), UNet items and launches per step, ms per UNet item, and whether the
graph latent equals the eager one bit for bit.  Then:
  - chunk sweep: DPM-Solver++ 20 at stride 8 with WINDOWS_PER_CHUNK in --chunks, ms per step and the sample's peak of
    torch.cuda.max_memory_allocated above what was allocated before it;
  - gather + merge alone: one step's gathers and merges captured in a CUDA graph and replayed between CUDA events.
The card name and power limit are read in the same run.
    python tools/panorama_bench.py [--rounds N] [--chunks 1,4,8,13,25]"""
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
from vdb200 import ops, parallel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--chunks", default="1,4,8,13,25")
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
H, W = 64, 256
xT = parallel.seeded_latents((0, 1), (4, H, W), seed=SEED).to(dev)
xT2 = parallel.seeded_latents((0, BS), (4, LAT, LAT), seed=SEED).to(dev)

# shared context buffers, as inpaint_bench.py does: the cross-attention layers keep one set of K / V^T projections per buffer, and
# alternating samplers replay their captured graphs instead of re-capturing them.  Config 2's [8, 77, 768] batch keeps its own.
ctx_bufs = {"config2": {}, "panorama": {}}


def make(cls, config2=False, **kw):
    s = cls(net, **kw)
    s._ctx_bufs = ctx_bufs["config2" if config2 else "panorama"]
    return s


def sample(smp, steps, stride):
    if stride is None:              # config 2
        x_info, shape, c, u = {"type": "image", "xt": xT2.clone()}, [BS, 4, LAT, LAT], c1.repeat(BS, 1, 1), u1.repeat(BS, 1, 1)
    else:
        x_info = {"type": "image", "xt": xT.clone(), "windows": panorama.Windows(64, stride)}
        shape, c, u = [1, 4, H, W], c1, u1
    return smp.sample(steps=steps, shape=shape, x_info=x_info, c_info={"type": "text", "conditioning": c,
                      "unconditional_conditioning": u, "unconditional_guidance_scale": SCALE}, verbose=False, eta=0.)[0]


SAMPLERS = {"ddim": (DDIMSampler, {}, 50), "dpmpp_2m": (DPMSolverSampler, {"order": 2}, 20)}
cases = [("config2_ddim_50", "ddim", None, True)]
for kind in SAMPLERS:
    for stride in (8, 16):
        for graph in (True, False):
            cases.append((f"{kind}_{SAMPLERS[kind][2]}_stride{stride}_{'graph' if graph else 'eager'}", kind, stride, graph))
samplers = {name: make(SAMPLERS[kind][0], config2=stride is None, use_cuda_graph=graph, **SAMPLERS[kind][1])
            for name, kind, stride, graph in cases}
e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def timed(name, kind, stride):
    torch.cuda.synchronize()
    e[0].record()
    x = sample(samplers[name], SAMPLERS[kind][2], stride)
    e[1].record()
    net.vae_decode(x, "image")
    e[2].record()
    torch.cuda.synchronize()
    return x, e[0].elapsed_time(e[1]), e[0].elapsed_time(e[2])


res = {name: {"call": [], "sample": []} for name, _, _, _ in cases}
with torch.no_grad():
    for name, kind, stride, _ in cases:          # warm-up: packs weights, captures each graph sampler's step graph
        for _ in range(2):
            timed(name, kind, stride)
        res[name]["launches_per_step"] = getattr(samplers[name], "last_step_launches", None)     # graph samplers count it
    for _ in range(args.rounds):
        for name, kind, stride, _ in cases:
            x, ms_sample, ms_call = timed(name, kind, stride)
            res[name]["call"].append(ms_call)
            res[name]["sample"].append(ms_sample)
            res[name]["x"] = x
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    net.vae_decode(res["ddim_50_stride8_graph"]["x"], "image")
    torch.cuda.synchronize()
    decode_peak_mb = (torch.cuda.max_memory_allocated() - base) / 2 ** 20

c2 = res["config2_ddim_50"]
c2_item = min(c2["sample"]) / 50 / (2 * BS)
for name, kind, stride, graph in cases:
    r = res[name]
    steps = SAMPLERS[kind][2]
    nwin = 1 if stride is None else panorama.layout(panorama.Windows(64, stride), H, W).nwin
    items = 2 * (BS if stride is None else nwin)
    out = dict(card=card, case=name, steps=steps, resolution="512x512 bs 4" if stride is None else "512x2048",
               ms_per_call=round(min(r["call"]), 2), ms_per_call_all=[round(v, 1) for v in r["call"]],
               ms_per_step=round(min(r["sample"]) / steps, 3), unet_items_per_step=items,
               launches_per_step=r["launches_per_step"], ms_per_unet_item=round(min(r["sample"]) / steps / items, 4),
               config2_ms_per_unet_item=round(c2_item, 4), finite=bool(torch.isfinite(r["x"]).all()))
    if stride is not None and graph:
        out["graph_equals_eager"] = bool(torch.equal(r["x"], res[name.replace("graph", "eager")]["x"]))
        out["windows"] = nwin
        out["windows_per_chunk"] = panorama.WINDOWS_PER_CHUNK
    print(json.dumps(out), flush=True)
print(json.dumps(dict(card=card, case="vae_decode_64x256_peak", peak_mb_above_allocated=round(decode_peak_mb, 1))), flush=True)

# ---- chunk sweep ----------------------------------------------------------------------------------------------------------------
for name in list(samplers):
    del samplers[name]
res = None
torch.cuda.synchronize()
torch.cuda.empty_cache()
default_chunk = panorama.WINDOWS_PER_CHUNK
with torch.no_grad():
    ref = None
    for per in [int(v) for v in args.chunks.split(",")]:
        panorama.WINDOWS_PER_CHUNK = per
        s = make(DPMSolverSampler, order=2)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        x = sample(s, 20, 8)                       # eager first step + capture + replays
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ms = []
        for _ in range(3):
            e[0].record()
            x = sample(s, 20, 8)
            e[1].record()
            torch.cuda.synchronize()
            ms.append(e[0].elapsed_time(e[1]))
        cos = 1.0 if ref is None else float(torch.nn.functional.cosine_similarity(x.flatten(), ref.flatten(), dim=0))
        ref = x if ref is None else ref
        print(json.dumps(dict(card=card, case="chunk_sweep_dpmpp_2m_20_stride8", windows_per_chunk=per,
                              ms_per_step=round(min(ms) / 20, 3), sample_peak_mb_above_allocated=round(peak, 1),
                              launches_per_step=s.last_step_launches, cos_to_first_chunk_size=round(cos, 6))), flush=True)

        # gather + merge alone, at this chunk size: one step's worth captured in a graph and replayed
        if per == default_chunk:
            st = s._st
            ws = st["regions"]                     # a panorama is the region walk with no regions
            lay = panorama.layout(panorama.Windows(64, 8), H, W)
            eps_in = torch.randn_like(ws.xw)

            def gm():
                for first, k in lay.chunks(per):
                    rows = 2 * k                       # [u block; c block] of n = 1
                    ops.region_gather(st["x_in"][:1], ws.oy, ws.ox, lay.h, lay.w, first, k, 0, 1, out=ws.xw[:rows])
                    ops.region_merge(eps_in[:rows], ws.oy, ws.ox, ws.cover_y, ws.cover_x, first, k, 0, None, ws.eps, halves=2)

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
            gm_ms = e[0].elapsed_time(e[1]) / reps
            print(json.dumps(dict(card=card, case="gather_merge_per_step_stride8", windows_per_chunk=per,
                                  ms_per_step=round(gm_ms, 4), launches=2 * len(lay.chunks(per)))), flush=True)
        del s
panorama.WINDOWS_PER_CHUNK = default_chunk
