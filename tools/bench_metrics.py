"""Times the per-frame PSNR / SSIM kernel (gcd_b200.metrics.frame_metrics -> gcd_frame_metrics) on the GPU.

    python tools/bench_metrics.py [--iters 200] [--reps 5] [--out results.json]

Workloads: 14 frames (one evaluation clip) at 256 x 384, the evaluation size, and at 576 x 1024, each with and without a mask.
The timed window is the kernel launch alone (the C entry point, which also zeroes the [frames, 8] output), over --iters launches
between two device events, after a warm-up of every workload; the workloads alternate within each of --reps repeats and the
median is reported. Image traffic is what the kernel must read once: pred and gt (2 x 4 B per pixel-channel) plus the 1 B mask per
pixel when there is one. Reports ms per call and GB/s of that traffic, with the card name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import ops  # noqa: E402
from gcd_b200._lib import check  # noqa: E402

T = 14


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metrics needs a GPU"
    res = {"card": card(), "torch": torch.__version__, "frames": T, "iters": a.iters, "reps": a.reps, "workloads": {}}
    print(res["card"], flush=True)
    lib = ops.lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    work = {}
    for H, W in ((256, 384), (576, 1024)):
        gt = torch.rand(T, 3, H, W, device="cuda", generator=g)
        pred = (gt + 0.02 * torch.randn(T, 3, H, W, device="cuda", generator=g)).clamp(0, 1)
        mask = (torch.rand(T, H, W, device="cuda", generator=g) > 0.3).to(torch.uint8)
        for masked in (False, True):
            m = mask if masked else None
            out = torch.empty(T, 8, device="cuda", dtype=torch.float64)
            nbytes = T * H * W * (3 * 8 + (1 if masked else 0))
            call = (lambda pred=pred, gt=gt, m=m, out=out, H=H, W=W:
                    check(lib.gcd_frame_metrics(ops._p(pred), ops._p(gt), ops._p(m), T, H, W, ops._p(out), ops._stream()),
                          "frame_metrics"))
            work[f"{H}x{W}" + ("_mask" if masked else "")] = (call, nbytes)
    for call, _ in work.values():
        for _ in range(10):
            call()
    torch.cuda.synchronize()
    times = {k: [] for k in work}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.reps):
        for name, (call, _) in work.items():
            e0.record()
            for _ in range(a.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters)
    for name, (_, nbytes) in work.items():
        ms = statistics.median(times[name])
        res["workloads"][name] = {"ms": ms, "ms_all": times[name], "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6}
        print(f"{name:>14}: {ms * 1e3:8.1f} us  {nbytes / ms / 1e6:7.1f} GB/s  (reps {', '.join(f'{t * 1e3:.1f}' for t in times[name])})",
              flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
