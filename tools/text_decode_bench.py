"""Optimus text decoding on one GPU at full size (12 layers, vocabulary 50260), synthetic weights, 4 rows (app.py's n_sample_text),
<EOS> never drawn so every row runs all 28 token steps.  Reports, from CUDA events after warm-up: ms per token step (replays of the
captured step graph), launches per step, and the bytes a step must read over its time against 3.35 TB/s (H100 SXM data sheet);
then one complete i2t call: 50 DDIM steps on the text latent, then the decode.  Prints the card name and power limit.
With --top-k / --top-p: ms per token step at 4 and 16 rows with the sampler's cuts off and on, the two graphs replayed
alternately in one session, and the launches per step of each.
With --num-beams K: 4 latents sampled (4 rows) against the same 4 latents under beam search (4 K rows, groups of 16 // K latents),
the two step graphs replayed alternately: ms per token step, launches per step and the time of a whole decode call of each.
    python tools/text_decode_bench.py [--no-i2t] [--top-k K] [--top-p P] [--num-beams K]"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ["VDB_TEXT_FLOWS"] = "1"
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))
import torch  # noqa: E402
from lib.cfg_helper import model_cfg_bank  # noqa: E402
from lib.model_zoo import get_model  # noqa: E402
from lib.model_zoo.ddim import DDIMSampler  # noqa: E402
from lib.model_zoo.optimus import STEPS_PER_CHECK  # noqa: E402
from vdb200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--no-i2t", action="store_true")
ap.add_argument("--top-k", type=int, default=0)
ap.add_argument("--top-p", type=float, default=0.0)
ap.add_argument("--num-beams", type=int, default=0)
args = ap.parse_args()
HBM = 3.35e12
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print("card:", card)
cfg = model_cfg_bank()('vd_four_flow_v1-0')
cfg.args.ctx_cfg_list = []
cfg.args.vae_cfg_list = [v for v in cfg.args.vae_cfg_list if v[0] == "text"]
t0 = time.time()
torch.manual_seed(0)
with torch.device(dev):
    net = get_model()(cfg, verbose=False)
g = torch.Generator(device=dev).manual_seed(1)
with torch.no_grad():
    for _, p in net.named_parameters():
        if p.ndim == 1 or not bool(p.any()):
            if p.ndim == 1 and p.shape[0] > 0 and bool((p == 1).all()):
                continue
            p.normal_(0.0, 0.02, generator=g)
net.eval()
net.to(dev)
vae = net.vae["text"]
print(f"built in {time.time() - t0:.1f} s")

R = 4
z = torch.randn(R, 768, generator=torch.Generator().manual_seed(3)).to(dev) * 3.0
with torch.no_grad():
    for _ in range(2):
        vae.decode_ids(z, eos_token=-1)                      # warm-up: packs weights, captures the step-chunk graph
    p = vae.packed()
    st = vae._state(R, dev)
    graph = st.graphs[(1.0, -1, 30, "seed", False, 0, 0.0, 0)]
    n0 = ops.launch_count()
    vae._step(st, p, 1.0, -1, 30, "seed", False)
    launches = ops.launch_count() - n0
    torch.cuda.synchronize()
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.step.zero_()
    e0.record()
    for i in range(reps):
        st.step.zero_()                                       # keep the step index inside the 28-step window
        st.done.zero_()                                       # the warm-up decodes left every row finished
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / (reps * STEPS_PER_CHECK)
    wbytes = sum(t.numel() * t.element_size() for L in p["layers"] for t in L.values() if torch.is_tensor(t))
    wbytes += sum(t.numel() * t.element_size() for L in p["layers"] for pair in (L["ln1"], L["ln2"]) for t in pair[:2])
    wbytes += p["lm_head"].numel() * 2 + R * 50260 * 4 * 2       # LM head weights, logits written then read by the sampler
    # one full decode call (28 steps, host checks every STEPS_PER_CHECK steps)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(5):
        vae.decode_ids(z, eos_token=-1)
    e1.record()
    torch.cuda.synchronize()
    ms_decode = e0.elapsed_time(e1) / 5
res = dict(card=card, rows=R, ms_per_token_step=round(ms_step, 4), launches_per_step=launches,
           bytes_per_step=wbytes, achieved_TBps=round(wbytes / (ms_step * 1e-3) / 1e12, 3),
           share_of_3_35_TBps=round(wbytes / (ms_step * 1e-3) / HBM, 3), ms_per_decode_28_steps=round(ms_decode, 3))
print(json.dumps(res))



def step_ms_off_and_on(R, top_k, top_p, rounds=5, reps=10):
    """ms per token step of the captured chunk with the cuts off and on, alternated over rounds; launches per step of each."""
    zr = torch.randn(R, 768, generator=torch.Generator().manual_seed(5)).to(dev) * 3.0
    cuts = {"off": (0, 0.0), "on": (top_k, top_p)}
    out = {}
    with torch.no_grad():
        st = vae._state(R, dev)
        for name, (k, p) in cuts.items():
            for _ in range(2):
                vae.decode_ids(zr, eos_token=-1, top_k=k, top_p=p)
            n0 = ops.launch_count()
            vae._step(st, vae.packed(), 1.0, -1, 30, "seed", False, k, p)
            out[name] = dict(launches_per_step=ops.launch_count() - n0, ms=[])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(rounds):
            for name, (k, p) in cuts.items():
                g = st.graphs[(1.0, -1, 30, "seed", False, k, p, 0)]
                e0.record()
                for _ in range(reps):
                    st.step.zero_()
                    st.done.zero_()
                    g.replay()
                e1.record()
                torch.cuda.synchronize()
                out[name]["ms"].append(e0.elapsed_time(e1) / (reps * STEPS_PER_CHECK))
    res = dict(card=card, rows=R, top_k=top_k, top_p=top_p)
    for name in cuts:
        res[f"ms_per_step_cuts_{name}"] = round(min(out[name]["ms"]), 4)
        res[f"ms_per_step_cuts_{name}_all"] = [round(v, 4) for v in out[name]["ms"]]
        res[f"launches_per_step_cuts_{name}"] = out[name]["launches_per_step"]
    res["filter_cost_share_of_step"] = round(res["ms_per_step_cuts_on"] / res["ms_per_step_cuts_off"] - 1.0, 4)
    return res


if args.top_k or 0.0 < args.top_p < 1.0:
    for rows_ in (4, 16):
        print(json.dumps(step_ms_off_and_on(rows_, args.top_k, args.top_p)))

def sampling_and_beams(K, n=4, rounds=5, reps=10):
    """ms per token step of sampling n latents (n rows) and of beam search over them (n K rows per group), the captured chunks
    replayed alternately; launches per step; one whole decode call of each (EOS never drawn: every step runs).  Before each timed chunk
    every row is re-armed (done = 0): a decode leaves all rows finished, and a finished row skips the sampler / beam-step work."""
    zr = torch.randn(n, 768, generator=torch.Generator().manual_seed(6)).to(dev) * 3.0
    per = 16 // K
    cases = {"sample": (n, "seed", 0, lambda: vae.decode_ids(zr, eos_token=-1)),
             "beam": (min(n, per) * K, "beam", K, lambda: vae.decode_beams(zr, K, eos_token=-1))}
    out = {}
    with torch.no_grad():
        for name, (rows, mode, k, call) in cases.items():
            for _ in range(2):
                call()
            st = vae._state(rows, dev)
            n0 = ops.launch_count()
            vae._step(st, vae.packed(), 1.0, -1, 30, mode, False, 0, 0.0, k)
            out[name] = dict(rows=rows, graph=st.graphs[(1.0, -1, 30, mode, False, 0, 0.0, k)], st=st,
                             launches_per_step=ops.launch_count() - n0, ms=[], ms_decode=[])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(rounds):
            for name, (rows, mode, k, call) in cases.items():
                o = out[name]
                torch.cuda.synchronize()
                e0.record()
                for _ in range(reps):
                    o["st"].step.zero_()
                    o["st"].done.zero_()          # a finished row would skip the sampler / beam work
                    o["graph"].replay()
                e1.record()
                torch.cuda.synchronize()
                o["ms"].append(e0.elapsed_time(e1) / (reps * STEPS_PER_CHECK))
                assert not bool(o["st"].done.any()), "a timed step ran on finished rows"
                e0.record()
                call()
                e1.record()
                torch.cuda.synchronize()
                o["ms_decode"].append(e0.elapsed_time(e1))
    res = dict(card=card, latents=n, num_beams=K, groups=-(-n // per))
    for name in cases:
        o = out[name]
        res[f"{name}_rows_per_step"] = o["rows"]
        res[f"{name}_ms_per_step"] = round(min(o["ms"]), 4)
        res[f"{name}_ms_per_step_all"] = [round(v, 4) for v in o["ms"]]
        res[f"{name}_launches_per_step"] = o["launches_per_step"]
        res[f"{name}_ms_per_decode"] = round(min(o["ms_decode"]), 3)
        res[f"{name}_ms_per_decode_all"] = [round(v, 3) for v in o["ms_decode"]]
    return res


if args.num_beams:
    print(json.dumps(sampling_and_beams(args.num_beams)))

if not args.no_i2t:
    bs = 4
    gq = torch.Generator().manual_seed(3)
    xT = torch.randn(bs, 768, generator=gq).to(dev)
    c = (torch.randn(bs, 257, 768, generator=gq) * 0.5).to(dev)
    u = torch.zeros(bs, 257, 768, device=dev)
    S = DDIMSampler(net)
    kw = dict(steps=50, shape=[bs, 768], x_info={"type": "text", "xt": xT},
              c_info={"type": "image", "conditioning": c, "unconditional_conditioning": u, "unconditional_guidance_scale": 7.5},
              verbose=False, eta=0.)
    with torch.no_grad():
        for _ in range(2):
            x, _ = S.sample(**{**kw, "x_info": {"type": "text", "xt": xT.clone()}})
            vae.decode_ids(x)                                 # the ids: no vocabulary file is needed to time the decode
        t_diff, t_dec = [], []
        for _ in range(3):
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            x, _ = S.sample(**{**kw, "x_info": {"type": "text", "xt": xT.clone()}})
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            rows = vae.decode_ids(x)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            t_diff.append((t2 - t1) * 1e3); t_dec.append((t3 - t2) * 1e3)
    print(json.dumps(dict(card=card, i2t_ms_diffusion_50_steps=round(min(t_diff), 2), i2t_ms_decode=round(min(t_dec), 2),
                          i2t_decode_tokens=[len(r) for r in rows])))
