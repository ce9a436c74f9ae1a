"""Tile sweep of the implicit-GEMM kernel over the long-K shapes of the UNet's 64x64 and 32x32 levels (bench.py c2 / c3): each
shape runs alone in a CUDA graph of 20 launches (as tools/bn_sweep.py does) with the tile forced, and the table prints TFLOP/s
per tile next to the tile's FLOP per operand byte loaded from L2 (BM * BN / (BM + BN)).  If the mainloop is
bound by the operand fill, TFLOP/s follows that column.  usage: python tools/igemm_tile_sweep.py"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "versatile-diffusion_b200"))
import torch
from vdb200 import ops

SHAPES = [  # (kind, dims, label)
    ("conv", (8, 64, 64, 320, 320), "3x3 B8 64x64 320->320"),
    ("conv", (8, 32, 32, 640, 640), "3x3 B8 32x32 640->640"),
    ("gemm", (32768, 320, 1280), "gemm M32768 N320 K1280"),
    ("gemm", (8192, 640, 2560), "gemm M8192 N640 K2560"),
]
TILES = [(128, 64), (128, 128), (128, 160), (128, 256), (256, 160)]


def time_graph(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    best = None
    for _ in range(5):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); g.replay(); e.record(); torch.cuda.synchronize()
        t = s.elapsed_time(e) / reps * 1000.0
        best = t if best is None else min(best, t)
    return best


q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True)
print("card: %s" % (q.stdout.strip() or torch.cuda.get_device_name()))
print("%-26s" % "tile (FLOP/B)" + "".join("  %4dx%-3d (%3.0f)" % (bm, bn, bm * bn / (bm + bn)) for bm, bn in TILES) + "      auto")
for kind, dims, label in SHAPES:
    if kind == "conv":
        B, H, W, C, N = dims
        x = torch.randn(B, H, W, C, device="cuda").bfloat16()
        w = (torch.randn(N, 9 * C, device="cuda") * 0.02).bfloat16()
        b = torch.randn(N, device="cuda")
        out = torch.empty(B, H, W, N, device="cuda", dtype=torch.bfloat16)
        flop = 2.0 * B * H * W * N * 9 * C
        run = lambda bn: ops.conv3x3(x, w, bias=b, out=out, bn=bn, ksplit=1 if bn else 0)
    else:
        M, N, K = dims
        a = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
        b = torch.randn(N, device="cuda")
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        flop = 2.0 * M * N * K
        run = lambda bn: ops.gemm(a, w, bias=b, resid=r, out=out, bn=bn, ksplit=1 if bn else 0)
    row = []
    for bm, bn in TILES + [(0, 0)]:
        forced = bn | (ops.BM256 if bm == 256 else 0)
        us = time_graph(lambda: run(forced))
        plan = ops.igemm_last_plan()
        row.append("  %6.1f us %5.1f" % (us, flop / us / 1e6))
        if not bn:
            row.append("  (%sx%d)" % (plan["bm"], plan["bn"]))
    print("%-26s" % label + "".join(row), flush=True)
