"""Times gcd_b200.infer's path on one clip, stage by stage, and gcd_frames_prepare against the reference's host cv2 stage.

    python tools/bench_infer.py [--reps 3] [--steps 25] [--samples 2] [--out results.json]

Workload: a seeded 14-frame 1920 x 1080 mp4 (mp4v, written here), --frame-stride 1, at GCD's 256 x 384 with --num_samples 2, 25
steps, the full-width Kubric UNet, decoder, conditioning encoder and ViT-H/14 tower with seeded weights (tools/bench_evaluate.py's
model). Stages: host decode (cv2.VideoCapture), upload + gcd_frames_prepare, conditioning, sampling (both samples in one run),
decode, writing (PNG folders and mp4s of input, predictions and uncertainty). Device stages are CUDA events, host stages a host
clock around work that ends in a device synchronise; one warm-up, then the best of --reps. The frame stage alone: the kernel on
device-resident frames (CUDA events, 50 launches) against the reference's host stage on the same decoded frames (u8 / 255,
center_crop_numpy, cv2.resize INTER_LINEAR per frame, `* 2 - 1`, `(x + 1) / 2`; host clock, best of 5). The card name and power
limit are read in the same run."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import infer as I, metrics, ops  # noqa: E402
from tools.bench_evaluate import build  # noqa: E402
from tools.bench_lpips import card  # noqa: E402

T, HW, SRC_HW = 14, (256, 384), (1080, 1920)


def write_clip(path):
    import cv2
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:SRC_HW[0], 0:SRC_HW[1]]
    w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 24.0, (SRC_HW[1], SRC_HW[0]))
    for t in range(T):
        img = np.stack([(xx + 8 * t) % 256, (yy + 4 * t) % 256, (xx + yy) // 12 % 256], -1).astype(np.uint8)
        w.write(np.clip(img.astype(np.int16) + rng.integers(-8, 9, img.shape), 0, 255).astype(np.uint8))
    w.release()


def host_cv2_stage(frames_bgr):
    """The reference's frame stage after decoding (common.load_video_mp4 + infer.py:137) on BGR -> RGB frames."""
    import cv2
    rgb = (frames_bgr[..., ::-1] / 255.0).astype(np.float32)
    y0, x0, ch, cw = I.crop_box(rgb.shape[1], rgb.shape[2], HW)
    rgb = rgb[:, y0:y0 + ch, x0:x0 + cw]
    rgb = np.stack([cv2.resize(x, (HW[1], HW[0]), interpolation=cv2.INTER_LINEAR) for x in rgb])
    return ((rgb * 2.0 - 1.0) + 1.0) / 2.0


def run_once(hot, args, path, out, S):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    g = I.example_generator(args.seed, 0, "cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    images, cmap = I.read_frames(path, I.clip_frames(T, 0, 1))
    t_decode = (time.perf_counter() - t0) * 1e3
    ev[0].record()
    input_rgb = I.prepare_frames(images, HW, True, cmap, "cuda")
    ev[1].record()
    batch = I.construct_batch("kubric", input_rgb, 30.0, 15.0, 0.0, 12, 127, 0.02, g)
    c, uc = hot.condition(batch)
    ev[2].record()
    rep = lambda d: {k: v.repeat(S, *([1] * (v.dim() - 1))) for k, v in d.items()}
    noise = torch.cat([torch.randn((T, 4, HW[0] // 8, HW[1] // 8), generator=g, device="cuda") for _ in range(S)])
    z = hot.sample_latents(noise, rep(c), rep(uc))
    ev[3].record()
    x = torch.cat([hot.decode_first_stage(z[s * T:(s + 1) * T], 14) for s in range(S)])
    sampled = torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0).view(S, T, 3, *HW)
    ev[4].record()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    unc, fd, md = metrics.sample_diversity(sampled)
    I.save_results(os.path.join(out, "extra", "bench_000_nseeded_clip"), input_rgb, sampled, unc, (fd, md), (6 + 12) // 2)
    t_write = (time.perf_counter() - t0) * 1e3
    return {"host_decode": t_decode, "upload_and_frames_prepare": ev[0].elapsed_time(ev[1]),
            "conditioning": ev[1].elapsed_time(ev[2]), "sampling": ev[2].elapsed_time(ev[3]), "decode": ev[3].elapsed_time(ev[4]),
            "writing": t_write}


def frame_stage(path):
    frames = I.read_video(path, list(range(T)))
    dev = frames.cuda()
    out = torch.empty(T, 3, *HW, device="cuda")
    box = I.crop_box(SRC_HW[0], SRC_HW[1], HW)
    ops.frames_prepare(dev, box, out, (2, 1, 0))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 50
    e0.record()
    for _ in range(n):
        ops.frames_prepare(dev, box, out, (2, 1, 0))
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / n
    np_frames = frames.numpy()
    host = []
    for _ in range(5):
        t0 = time.perf_counter()
        ref = host_cv2_stage(np_frames)
        host.append((time.perf_counter() - t0) * 1e3)
    err = np.abs(out.cpu().numpy().transpose(0, 2, 3, 1).astype(np.float64) - ref).max()
    return {"frames_prepare_kernel_ms": kernel_ms, "reference_host_cv2_ms": min(host), "speedup": min(host) / kernel_ms,
            "max_abs_diff_vs_host_cv2": float(err), "cv2_ipp": bool(__import__("cv2").ipp.useIPP())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--samples", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer measures on a CUDA device")
    hot, _ = build(a.steps)
    args = I.parser().parse_args(["--kind", "kubric", "--checkpoint", "seeded", "--input", "clip.mp4", "--output", "out"])
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "clip_1080p.mp4")
        write_clip(path)
        run_once(hot, args, path, os.path.join(tmp, "out"), a.samples)
        runs = [run_once(hot, args, path, os.path.join(tmp, "out"), a.samples) for _ in range(a.reps)]
        frames = frame_stage(path)
    best = {k: min(r[k] for r in runs) for k in runs[0]}
    res = {"workload": f"one {T}-frame {SRC_HW[1]}x{SRC_HW[0]} mp4 -> {HW[0]} x {HW[1]}, {a.samples} samples, {a.steps} steps, "
                       "full-width Kubric UNet", "stage_ms": best, "total_ms": sum(best.values()), "all_runs": runs,
           "frame_stage": frames, "card": card()}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
