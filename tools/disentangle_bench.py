"""Time the image-context rank adjustment (app.py's adjust_rank, q = 20, niter = 100) on the GPU: the one-launch kernel
(lib.model_zoo.disentangle.adjust_rank) beside the torch path app.py runs (torch.linalg.qr / svd through the oracle at fp32 on the
device, which is what torch.pca_lowrank does).  Needs a CUDA device; prints one JSON line per batch size, with the card's name and
power limit read in the same run.

    python tools/disentangle_bench.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "versatile-diffusion_b200")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("disentangle_bench: needs a CUDA device")
    from lib.model_zoo.disentangle import adjust_rank
    from oracle.disentangle_oracle import rank_adjust as torch_path
    from vdb200 import ops
    name = card()
    ar = adjust_rank()
    lvl = 0.25
    f = ar.factors(lvl)
    for n in (1, 4):
        x = torch.randn(n, 256, 768, device="cuda", generator=torch.Generator("cuda").manual_seed(n))
        R = torch.randn(256, 20, device="cuda")
        kernel = time_ms(lambda: ar(x, lvl, R=R), args.iters, args.warmup)
        ref = time_ms(lambda: torch_path(x, R, f, True, dtype=torch.float32), max(2, args.iters // 4), 1)
        ops.reset_launch_count()
        ar(x, lvl, R=R)
        torch.cuda.synchronize()
        launches = ops.launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch_path(x, R, f, True, dtype=torch.float32)
            torch.cuda.synchronize()
        ref_launches = sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)
        err = (ar(x, lvl, R=R) - torch_path(x, R, f, True, dtype=torch.float64)[0].float()).abs().max().item()
        print(json.dumps(dict(n=n, m=256, q=20, niter=100, kernel_ms=round(kernel, 4), kernel_launches=launches,
                              torch_path_ms=round(ref, 3), torch_path_kernels=ref_launches, max_abs_err_vs_fp64=err, card=name)))


if __name__ == "__main__":
    main()
