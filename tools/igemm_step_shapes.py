"""Where the implicit-GEMM time of one DDIM step goes, per launch shape.

Records the GEMM / conv launches (igemm_kernel: every conv and linear layer of the UNet) of one eager DDIM step of a bench.py
config (ops.record_start / record_stop), groups them by shape and kernel plan, and replays each group alone inside a CUDA graph
(--copies back-to-back copies per graph, so the graph launch is amortised), timed with CUDA events, best of --reps.  Prints per
group: launches per step, us per step, TFLOP/s, share of the whole step (the CUDA-graph step of the sampler, timed the same way)
and the plan (BM, BN, STAGES, MODE, ksplit, grid), with the card's name and power limit.  A group replayed alone runs with a warmer
L2 than inside the step, so the per-group times are a lower bound on what the same launches cost there.

VDB200_LIB=<other libvdb200.so> times another build of the kernels on the same shapes; --json writes the rows, and --baseline
<rows of another run> adds its times and the change per group.

    python tools/igemm_step_shapes.py [--config c2] [--reps 5] [--copies 10] [--json out.json] [--baseline old.json]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))

import torch  # noqa: E402

import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def describe(fn, cargs, flops):
    """shape of one recorded launch (argument order of ops.gemm / ops.gemm_ln / ops.conv3x3)"""
    name = fn.__name__
    if name == "vdb_gemm_bf16":
        M, K, N = cargs[1], cargs[2] + cargs[5], cargs[8]
        extra = "".join([" act%d" % cargs[18] if cargs[18] else "", " +resid" if cargs[13] else ""])
        return "gemm M%d N%d K%d%s" % (M, N, K, extra)
    if name == "vdb_gemm_ln_bf16":
        M, K, N = cargs[1], cargs[2], cargs[5]
        kind = " ln-in" if cargs[13] else " stats-out"
        extra = "".join([" act%d" % cargs[12] if cargs[12] else "", " +resid" if cargs[8] else ""])
        return "gemm_ln M%d N%d K%d%s%s" % (M, N, K, kind, extra)
    B, H, W, C, mode, N = cargs[1], cargs[2], cargs[3], cargs[4], cargs[5], cargs[7]
    M = B * (H // 2) * (W // 2) if mode in (1, 2) else B * H * W
    K = round(flops / 2.0 / N / M)
    return "conv3x3 mode%d B%d %dx%d C%d N%d (M%d K%d)%s" % (mode, B, H, W, C, N, M, K, " +resid" if cargs[15] else "")


def time_graph(run, reps):
    """best of `reps` CUDA-event timings (ms) of a graph that calls run() once"""
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    g.replay()
    torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1)
        best = t if best is None else min(best, t)
    del g
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c2", choices=sorted(bench.CONFIGS))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--copies", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--baseline", default=None)
    args = ap.parse_args()

    from lib.model_zoo.ddim import DDIMSampler
    from vdb200 import _lib, ops

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card: %s   library: %s" % (card(), _lib.LIB_PATH))
    net = bench.build_net(dev)
    cfg = bench.CONFIGS[args.config]
    g = torch.Generator().manual_seed(2)
    ctxs = []
    for ctype, L, ratio in cfg["ctx"]:
        c = torch.randn(1, L, 768, generator=g) * 0.5
        u = torch.zeros(1, L, 768) if ctype == "image" else torch.randn(1, L, 768, generator=g) * 0.5
        ctxs.append((ctype, ratio, c.to(dev).repeat(bench.BS, 1, 1), u.to(dev).repeat(bench.BS, 1, 1)))
    xT = torch.randn(bench.BS, 4, bench.LAT, bench.LAT, generator=torch.Generator().manual_seed(bench.SEED)).to(dev)
    shape = [bench.BS, 4, bench.LAT, bench.LAT]

    def sample(smp, steps):
        xi = {"type": "image", "xt": xT}
        if len(ctxs) == 1:
            t, _, c, u = ctxs[0]
            return smp.sample(steps=steps, shape=shape, x_info=xi, verbose=False, eta=0.,
                              c_info={"type": t, "conditioning": c, "unconditional_conditioning": u,
                                      "unconditional_guidance_scale": bench.SCALE})[0]
        return smp.sample_multicontext(steps=steps, shape=shape, x_info=xi, verbose=False, eta=0.,
                                       c_info_list=[{"type": t, "conditioning": c, "unconditional_conditioning": u,
                                                     "unconditional_guidance_scale": bench.SCALE, "ratio": r}
                                                    for t, r, c, u in ctxs])[0]

    with torch.no_grad():
        # the whole step: the sampler's own CUDA-graph path, 10 steps, per step
        graphed = DDIMSampler(net)
        sample(graphed, 10)
        torch.cuda.synchronize()
        best_step = None
        for _ in range(max(args.reps // 2, 2)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            sample(graphed, 10)
            e1.record()
            torch.cuda.synchronize()
            t = e0.elapsed_time(e1) / 10
            best_step = t if best_step is None else min(best_step, t)
        del graphed

        eager = DDIMSampler(net, use_cuda_graph=False)
        sample(eager, 1)
        ops.record_start()
        sample(eager, 1)
        recs = ops.record_stop()
        torch.cuda.synchronize()

        groups, key_plans = OrderedDict(), {}
        for rec in recs:
            fn, cargs, _keep, flops = rec
            ops.check(fn(*cargs, ops._stream()), "igemm_step_shapes")
            plan = ops.igemm_last_plan()
            # (the key is the shape alone, so that --baseline lines a group up with a build that plans it differently)
            key = describe(fn, cargs, flops)
            tile = "BM %d BN %d ST %d MODE %d ks %d grid %d" % (plan["bm"], plan["bn"], plan["stages"], plan["mode"],
                                                                plan["ksplit"], plan["grid"])
            key_plans.setdefault(key, tile)
            grp = groups.setdefault(key, {"recs": [], "flops": 0.0})
            grp["recs"].append(rec)
            grp["flops"] += flops
        torch.cuda.synchronize()

        rows = []
        for key, grp in groups.items():
            def run(grp=grp):
                for _ in range(args.copies):
                    ops.replay(grp["recs"])
            ms = time_graph(run, args.reps) / args.copies
            rows.append({"key": key, "plan": key_plans[key], "launches": len(grp["recs"]), "us": ms * 1e3,
                         "tflops": grp["flops"] / ms / 1e9})
        all_ms = time_graph(lambda: ops.replay(recs), args.reps)

    base = {}
    if args.baseline:
        base = {r["key"]: r for r in json.load(open(args.baseline))["rows"]}
    tot = sum(r["us"] for r in rows)
    print("config %s: one DDIM step (CUDA graph) %.3f ms; its %d igemm launches replayed together %.3f ms, group by group %.3f ms"
          % (args.config, best_step, len(recs), all_ms, tot / 1e3))
    hdr = "%9s %7s %5s %6s  %s" % ("us/step", "TFLOP/s", "n", "step%", "shape | plan")
    if base:
        hdr = "%9s %7s " % ("base us", "change") + hdr
    print(hdr)
    for r in sorted(rows, key=lambda r: -r["us"]):
        line = "%9.1f %7.1f %5d %5.1f%%  %s | %s" % (r["us"], r["tflops"], r["launches"], 100.0 * r["us"] / 1e3 / best_step, r["key"],
                                                      r["plan"])
        if base:
            b = base.get(r["key"])
            line = ("%9.1f %+6.1f%% " % (b["us"], 100.0 * (r["us"] / b["us"] - 1)) if b else "%9s %7s " % ("-", "-")) + line
            if b and b.get("plan") != r["plan"]:
                line += "   (baseline: %s)" % b.get("plan")
        print(line)
    if base:
        bt = sum(b["us"] for b in base.values())
        print("sum over groups: %.1f us, baseline %.1f us (%+.1f%%)" % (tot, bt, 100.0 * (tot / bt - 1)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "config": args.config, "step_ms": best_step, "igemm_all_ms": all_ms, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
