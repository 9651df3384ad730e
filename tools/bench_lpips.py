"""Times LPIPS over one evaluation example on the GPU: the CUDA path (gcd_b200.lpips) against the fp32 torch restatement of the
reference (oracle/lpips_oracle.py, cuDNN without TF32) on the same GPU.

    python tools/bench_lpips.py [--reps 3] [--out results.json]

Workload: one example of gcd-model/scripts/test.py (14 ground-truth frames, 2 samples of 14 frames, --num_samples default 2) scored
as metrics.frame_lpips does it: the ground truth's features once, 28 (sample, ground truth) pairs; at 256 x 384 and at 576 x 1024.
The oracle runs the reference's order (VGG16 of both frames for every pair), in chunks of 7 pairs. Weights are the seeded ones of the
goldens (oracle/lpips_oracle.seeded_state), inputs seeded smooth fields. Device events, one warm-up of each path, then the two
paths alternate. Reports ms per example and TFLOP/s from shape-computed FLOPs (2 x MAC of the 13 convs, the frames each path
actually runs), a per-op breakdown of one CUDA pass (ops.profile, a separate run), the agreement with the oracle, and the card
name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import metrics, ops  # noqa: E402
from gcd_b200.lpips import LPIPS, SLICES  # noqa: E402
from oracle import lpips_oracle as O  # noqa: E402

S, T = 2, 14


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def conv_flops(H, W):
    """2 x MAC of VGG16's 13 convolutions for one H x W frame, per conv, with the pooled sizes."""
    out, h, w, cin = [], H, W, 3
    for k, (idx, cout) in enumerate(zip(SLICES, O.CHNS)):
        if k > 0:
            h, w = h // 2, w // 2
        for _ in idx:
            out.append(2.0 * h * w * cout * cin * 9)
            cin = cout
    return out


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="256x384,576x1024")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lpips needs a GPU"
    dev = "cuda:0"
    res = {"card": card(), "torch": torch.__version__, "act_dtype": str(ops.act_dtype()), "samples": S, "frames": T}
    print(res["card"], flush=True)
    sd = O.seeded_state(0)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    model = LPIPS()
    model.load_state_dict(sd)
    for size in a.sizes.split(","):
        H, W = (int(v) for v in size.split("x"))
        pred, gt = O.pair_inputs(S * T, H, W, seed=H)
        pred = ((pred.view(S, T, 3, H, W) + 1) / 2).to(dev)
        gt = ((gt[:T] + 1) / 2).to(dev)

        def cuda():
            return metrics.frame_lpips(pred, gt, model)

        def oracle():
            x, y = pred.reshape(S * T, 3, H, W) * 2 - 1, (gt * 2 - 1).repeat(S, 1, 1, 1)
            return torch.cat([O.lpips(sd_dev, y[i:i + 7], x[i:i + 7]) for i in range(0, S * T, 7)]).view(S, T).double().cpu()

        _, oc = timed(cuda)
        _, oo = timed(oracle)
        tc, to = [], []
        for _ in range(a.reps):
            tc.append(timed(cuda)[0])
            to.append(timed(oracle)[0])
        with ops.profile() as prof:
            ops.DETAIL = True
            cuda()
            ops.DETAIL = False
        per_op = {k: round(v["ms"], 4) for k, v in prof.summary().items()}
        per_frame = conv_flops(H, W)
        fl_cuda = sum(per_frame) * (T + S * T)
        fl_oracle = sum(per_frame) * 2 * S * T
        ms_c, ms_o = min(tc), min(to)
        n64 = per_frame[0] + per_frame[1]
        ms64 = sum(v for k, v in per_op.items() if k.startswith("tc ") and " N64 " in k)
        d = (oc - oo).abs()
        r = {"ms_cuda": ms_c, "ms_cuda_all": tc, "ms_torch_oracle": ms_o, "ms_torch_oracle_all": to, "speedup": ms_o / ms_c,
             "tflop_cuda": fl_cuda / 1e12, "tflops_cuda": fl_cuda / ms_c / 1e9, "tflop_oracle": fl_oracle / 1e12,
             "tflops_oracle": fl_oracle / ms_o / 1e9, "n64_flop_share": n64 / sum(per_frame), "n64_ms": ms64,
             "per_op_ms": per_op, "agreement": {"max_abs": d.max().item(), "rel_l2": ((oc - oo).norm() / oo.norm()).item()}}
        res[f"{H}x{W}"] = r
        print(size, json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
