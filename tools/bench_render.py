"""Times the point-cloud view synthesis of one evaluation example on the GPU: the CUDA path (gcd_b200.render) against the torch
restatement of the reference's renderer (oracle/render_oracle.py) run on the same GPU, as the reference runs it on its data GPU.

    python tools/bench_render.py [--reps 3] [--out results.json]

Workloads (14 frames, 280 x 420 renders resized to 256 x 384, spread radius 1):
  kubric  16 views of 384 x 576 points per frame (the 576 / 384 aspect synth_src_dst_rgb corrects for; convert_pcl_kubric.py stores
          one point per pixel), src + dst at blur 21 and the view-4 reprojection at blur 3: 3 renders per frame;
  pardom  19 views of 480 x 640 points per frame, the segm modality with modal_time 0 at blur 21 and the view-16 reprojection: 2 renders.
Clouds are seeded synthetic scenes (render_oracle.synthetic_clouds); to keep set-up short two distinct frames are generated and
repeated over the 14 (the cost does not depend on which frame it is). Device events after one warm-up of each path; the two paths
alternate. Reports ms per example, points per second and the output agreement, with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import render  # noqa: E402
from oracle import render_oracle as O  # noqa: E402

T = 14


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def clip(kind, V, h, w, seed):
    cl = O.synthetic_clouds(kind, 2, V, h, w, seed)
    idx = torch.arange(T) % 2
    return {k: (v[idx] if k in ("xyz", "rgb", "segm", "intrinsics") else v) for k, v in cl.items()}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def agreement(a, b):
    d = torch.cat([(x - y).abs().flatten() for x, y in zip(a, b)])
    return {"max_abs": d.max().item(), "frac_within_1e-5": (d <= 1e-5).double().mean().item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_render needs a GPU"
    res = {"card": card(), "torch": torch.__version__, "frames": T, "render_hw": [280, 420], "frame_hw": [256, 384]}
    print(res["card"], flush=True)

    kc = clip("kubric", 16, 384, 576, 41)
    kx, kr = kc["xyz"].cuda(), kc["rgb"].cuda()
    src, dst = O.trajectory(T, 10, 50, 14, 3).cuda(), O.trajectory(T, 100, 160, 13, 4).cuda()
    pc = clip("pardom", 19, 480, 640, 42)
    px, pr, ps, pal = pc["xyz"].cuda(), pc["rgb"].cuda(), pc["segm"].cuda(), pc["palette"].cuda()
    pe = O.trajectory(T, 16 / 19 * 360 - 10, 16 / 19 * 360 + 10, 14, 3).cuda()
    work = {
        "kubric": dict(points=T * (2 * 16 + 1) * 384 * 576, renders=3 * T,
                       cuda=lambda: render.kubric_views(kx, kr, kc["intrinsics"][0], src, dst, True),
                       oracle=lambda: O.kubric_views(kx, kr, kc["intrinsics"][0], src, dst, True)),
        "pardom": dict(points=T * (19 + 1) * 480 * 640, renders=2 * T,
                       cuda=lambda: render.pardom_views(px, pr, pc["intrinsics"], pe, "segm", ps, pal, 0, True),
                       oracle=lambda: O.pardom_views(px, pr, pc["intrinsics"], pe, "segm", ps, pal, 0, True)),
    }
    for name, w in work.items():
        _, oc = timed(w["cuda"])
        _, oo = timed(w["oracle"])
        tc, to = [], []
        for _ in range(a.reps):
            tc.append(timed(w["cuda"])[0])
            to.append(timed(w["oracle"])[0])
        ms_c, ms_o = min(tc), min(to)
        r = {"ms_cuda": ms_c, "ms_cuda_all": tc, "ms_torch_oracle": ms_o, "ms_torch_oracle_all": to, "speedup": ms_o / ms_c,
             "point_renders": w["points"], "renders": w["renders"], "points_per_s_cuda": w["points"] / ms_c * 1e3,
             "points_per_s_oracle": w["points"] / ms_o * 1e3,
             "agreement": agreement([x for x in oc if x is not None], [x.to(oc[0].device) for x in oo if x is not None])}
        res[name] = r
        print(name, json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
