"""Time every attention launch shape of a c2 / c3 DDIM step, each alone in a CUDA graph.

The UNet of bench.py runs, at B 8 (the CFG pair of a batch of four) and 8 heads, self-attention at the 64x64, 32x32 and 16x16
latent levels (N 4096 d_head 40, N 1024 d_head 80, N 256 d_head 160) and cross-attention at the same levels over the 77 text
tokens (c2) or the 257 CLIP image tokens (c3).  Each shape is launched --copies times back to back inside one CUDA graph (so
the graph launch is amortised), timed with CUDA events, best of --reps.  Prints per shape: us per launch, useful TFLOP/s
(4 B H Nq Nk d_head) and the share of the MUFU-only bound, B H Nq Nk / (16 ex2 per clock per SM x SMs x the card's maximum SM
clock): one MUFU ex2 per score is what the softmax would need without the polynomial exponentials, so a share near 100% means
the launch runs as fast as the special-function units alone would allow.  Prints the card's name and power limit first.

VDB200_LIB=<other libvdb200.so> times another build of the kernels; --json writes the rows, and --baseline <rows of another
run> adds its times and the change per shape.

    python tools/attention_shapes.py [--reps 20] [--copies 20] [--json out.json] [--baseline old.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.join(ROOT, "versatile-diffusion_b200"))

import torch  # noqa: E402

from igemm_step_shapes import card, time_graph  # noqa: E402

B, H = 8, 8
# (name, Nq, Nk, d_head); Nk == Nq is self-attention through the fused q | k projection output
SHAPES = [("self", 4096, 4096, 40), ("self", 1024, 1024, 80), ("self", 256, 256, 160)]
SHAPES += [("cross", n, L, d) for L in (77, 257) for n, d in ((4096, 40), (1024, 80), (256, 160))]


def max_sm_clock_hz():
    q = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return float(q.stdout.strip()) * 1e6


def launcher(ops, kind, Nq, Nk, d):
    """inputs laid out as lib/model_zoo/attention.py lays them out; returns a function that runs the launch once"""
    dk, dv = ops.attention_pads(d)
    g = torch.Generator(device="cuda").manual_seed(Nq * 1000 + Nk + d)

    def rnd(*shape):
        return (torch.randn(*shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16)
    out = torch.empty(B * Nq, H * d, dtype=torch.bfloat16, device="cuda")
    if kind == "self":
        qk, vt = rnd(B * Nq, 2 * H * dk), rnd(H * dv, B * Nq)
        return lambda: ops.attention(qk, qk, vt, out, B, H, Nq, Nq, d, q_col0=0, k_col0=H * dk)
    Lp = (Nk + 7) // 8 * 8
    q, k, vt = rnd(B * Nq, H * dk), rnd(B * Lp, H * dk), rnd(H * dv, B * Lp)
    return lambda: ops.attention(q, k, vt, out, B, H, Nq, Nk, d, kv_bstride=Lp)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--copies", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--baseline", default=None)
    args = ap.parse_args()

    from vdb200 import _lib, ops

    torch.cuda.set_device(0)
    name = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clock = max_sm_clock_hz()
    print("card: %s   library: %s" % (name, _lib.LIB_PATH))
    rows = []
    with torch.no_grad():
        for kind, Nq, Nk, d in SHAPES:
            run = launcher(ops, kind, Nq, Nk, d)

            def copies(run=run):
                for _ in range(args.copies):
                    run()
            run()
            ms = time_graph(copies, args.reps) / args.copies
            mufu_ms = B * H * Nq * Nk / (16.0 * sms * clock) * 1e3
            rows.append({"key": "%s B%d H%d Nq %d Nk %d d %d" % (kind, B, H, Nq, Nk, d), "us": ms * 1e3,
                         "tflops": 4.0 * B * H * Nq * Nk * d / ms / 1e9, "mufu_share": mufu_ms / ms})

    base = {}
    if args.baseline:
        base = {r["key"]: r for r in json.load(open(args.baseline))["rows"]}
    print("MUFU bound at %d SMs x %.0f MHz" % (sms, clock / 1e6))
    hdr = "%9s %7s %6s  %s" % ("us", "TFLOP/s", "MUFU%", "shape")
    if base:
        hdr = "%9s %7s " % ("base us", "change") + hdr
    print(hdr)
    for r in rows:
        line = "%9.1f %7.1f %5.1f%%  %s" % (r["us"], r["tflops"], 100.0 * r["mufu_share"], r["key"])
        if base:
            b = base.get(r["key"])
            line = ("%9.1f %+6.1f%% " % (b["us"], 100.0 * (r["us"] / b["us"] - 1)) if b else "%9s %7s " % ("-", "-")) + line
        print(line)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "library": _lib.LIB_PATH, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
