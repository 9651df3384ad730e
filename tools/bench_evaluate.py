"""Times one Kubric-4D evaluation example on the GPU: gcd_b200.evaluate.evaluate_example (conditioning once, the S samples as S clips
of one sampler run) against the reference's shape (scripts/test.py run_inference: S sequential sample_video calls, each
re-running the conditioner), both followed by the same calculate_metrics.

    python tools/bench_evaluate.py [--reps 3] [--steps 25] [--samples 2] [--out results.json]

Workload: GCD's evaluation settings, 14 frames at 256 x 384 (latent 32 x 48), --num_samples 2, 25 steps, the full-width Kubric UNet
(spec.UNET_KUBRIC), decoder, conditioning encoder and ViT-H/14 tower with seeded weights (gcd_b200.synthetic), LPIPS with the
seeded weights of the goldens; the example's views are rendered once from a synthetic point cloud. Each path is warmed up once,
then the two alternate `--reps` times; the best time of each is reported (host clock around work that ends in a device
synchronise), with the rel-L2 agreement of the two paths' latents and the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import clip, evaluate as E, metrics, render, spec, synthetic  # noqa: E402
from gcd_b200.lpips import LPIPS  # noqa: E402
from gcd_b200.pipeline import GCDHotPath  # noqa: E402
from oracle import lpips_oracle as LO, render_oracle as RO  # noqa: E402
from tools.bench_lpips import card  # noqa: E402

T, HW, RENDER_HW = 14, (256, 384), (280, 420)


def build(steps):
    hot = GCDHotPath(spec.UNET_KUBRIC, spec.VAE_DECODER, num_steps=steps, num_frames=T, device="cuda")
    hot.load_state(synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_KUBRIC), seed=0),
                   synthetic.seeded_state(spec.decoder_param_shapes(spec.VAE_DECODER), seed=0))
    shapes = dict(clip.TEXT_LEFTOVERS_H14, **{"visual." + k: v for k, v in clip.visual_param_shapes(clip.VIT_H14).items()})
    hot.load_clip({"model." + k: v for k, v in synthetic.seeded_state(shapes, seed=1).items()})
    q = synthetic.seeded_state({"w": (8, 8, 1, 1), "b": (8,)}, seed=2)
    hot.load_cond_encoder(synthetic.seeded_state(spec.encoder_param_shapes(spec.VAE_ENCODER), seed=2), q["w"], q["b"])
    sp = synthetic.seeded_state({"proj.weight": (128, 13), "proj.bias": (128,)}, seed=3)
    hot.load_spherical(sp["proj.weight"], sp["proj.bias"])
    lp = LPIPS()
    lp.load_state_dict(LO.seeded_state(0))
    return hot, lp.cuda()


def example():
    cl = RO.synthetic_clouds("kubric", T, 16, 96, 144, 7)
    traj = E.kubric_trajectories(E.control_row("kubric", None, 0, 2, 12, (20.0, 30.0, 10.0, 15.0, 15.0, 0.0)))
    src, dst, rep = render.kubric_views(cl["xyz"].cuda(), cl["rgb"].cuda(), cl["intrinsics"][0], traj["extrinsics_src"],
                                        traj["extrinsics_dst"], True, RENDER_HW, HW)
    batch = E.construct_batch("kubric", traj, src, dst, rep, 12, torch.Generator(device="cuda").manual_seed(7))
    return (batch["jpg"], batch["reproject"]), batch


def batched(hot, lp, views, batch, S):
    samples, m, _ = E.evaluate_example(hot, views, batch, S, torch.Generator(device="cuda").manual_seed(11), lpips=lp)
    return torch.cat([s["sampled_latent"] for s in samples]), m


def sequential(hot, lp, views, batch, S):
    g = torch.Generator(device="cuda").manual_seed(11)
    zs, xs = [], []
    for _ in range(S):
        c, uc = hot.condition(batch)
        z, x = hot.sample_video(torch.randn((T, 4, HW[0] // 8, HW[1] // 8), generator=g, device="cuda"), c, uc)
        zs.append(z)
        xs.append(torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0))
    m, _ = metrics.calculate_metrics((views[0] + 1.0) / 2.0, (views[1] + 1.0) / 2.0, torch.stack(xs), lpips=lp)
    return torch.cat(zs), m


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--samples", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate measures on a CUDA device")
    hot, lp = build(a.steps)
    views, batch = example()
    paths = {"batched": lambda: batched(hot, lp, views, batch, a.samples),
             "sequential": lambda: sequential(hot, lp, views, batch, a.samples)}
    for fn in paths.values():
        timed(fn)
    times = {k: [] for k in paths}
    outs = {}
    for _ in range(a.reps):
        for k, fn in paths.items():
            ms, outs[k] = timed(fn)
            times[k].append(ms)
    zb, zs = outs["batched"][0], outs["sequential"][0]
    best = {k: min(v) for k, v in times.items()}
    res = {"workload": f"Kubric example, {T} x {HW[0]} x {HW[1]}, {a.samples} samples, {a.steps} steps, full-width UNet, metrics + LPIPS",
           "ms_per_example": best, "all_ms": times, "speedup": best["sequential"] / best["batched"],
           "latent_rel_l2_batched_vs_sequential": ((zb - zs).norm() / zs.norm()).item(),
           "mean_psnr": {k: outs[k][1]["mean_psnr"].tolist() for k in paths}, "card": card()}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
