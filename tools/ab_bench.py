"""A/B of two builds of libgcd_b200.so on one GPU, in one process tree: bench.py alternating old / new, then the outputs compared.

    python tools/ab_bench.py --old <old .so> [--new <new .so>] [--reps 3] [--steps 3] [--warmup 3] [--out <summary .json>]

Each run is `bench.py --gpus 1 --no-cpu-baseline --dump-outputs <dir>` with GCD_LIB_PATH selecting the library (README,
environment switches); the first run of each library also measures the extra workloads, the others pass --no-extra.
Prints the card and its power limit, each run's value / ms_per_step / tc_gemm TFLOP/s / gpu_launches, mean and spread
(max - min) per library, and the rel-L2 of the dumped latents and frames old-vs-new and old-vs-old. Alternating the two in one
call is what makes the difference comparable with the spread: other work shares the host, and clocks drift.
"""
import argparse
import json
import os
import subprocess
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(lib, out_dir, args, extra):
    env = dict(os.environ)
    if lib:
        env["GCD_LIB_PATH"] = os.path.abspath(lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--no-cpu-baseline", "--dump-outputs", out_dir] + ([] if extra else ["--no-extra"])
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        sys.exit(f"bench.py failed with {lib}:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    for ln in reversed(r.stdout.splitlines()):
        if ln.startswith("{") and '"value"' in ln:
            return json.loads(ln)
    sys.exit(f"no result line from bench.py with {lib}:\n{r.stdout[-2000:]}")


def rel_l2(a_dir, b_dir):
    out = {}
    for name in ("latents", "frames_stride2"):
        a, b = (np.load(os.path.join(d, name + ".npy")).astype(np.float64) for d in (a_dir, b_dir))
        out[name] = float(np.linalg.norm(a - b) / (np.linalg.norm(a) + 1e-30))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--old", required=True)
    ap.add_argument("--new", default=None, help="default: the in-tree build")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the summary and every run's result line to this JSON file")
    args = ap.parse_args()
    dumps = tempfile.mkdtemp(prefix="gcd_ab_")          # the dumped arrays (25 MB of frames per run) are compared, not kept
    res = {"old": [], "new": []}
    for i in range(args.reps):
        for which, lib in (("old", args.old), ("new", args.new)):
            line = run(lib, os.path.join(dumps, f"{which}{i}"), args, extra=(i == 0))
            res[which].append(line)
            if i == 0 and which == "old":
                print("card:", json.dumps(line.get("gpu")), flush=True)
            print(f"{which} run {i}: value {line['value']} latent-frames/s  ms_per_step {line['ms_per_step']}  "
                  f"tc_gemm {line['roofline']['achieved']} TFLOP/s  e2e {line['e2e']['value']}  gpu_launches {line['gpu_launches']}", flush=True)
            if "extra_workloads" in line:
                print(f"{which} extra_workloads: {json.dumps(line['extra_workloads'])}", flush=True)
    summary = {}
    for which, lines in res.items():
        v = [ln["value"] for ln in lines]
        summary[which] = {"mean": sum(v) / len(v), "spread": max(v) - min(v), "values": v}
        print(f"{which}: mean {summary[which]['mean']:.4f}  spread {summary[which]['spread']:.4f}  {v}")
    gain = summary["new"]["mean"] / summary["old"]["mean"] - 1
    noise = max(summary["old"]["spread"], summary["new"]["spread"]) / summary["old"]["mean"]
    print(f"new vs old: {100 * gain:+.2f} %  (largest spread {100 * noise:.2f} % of the old mean)")
    summary["rel_l2_old_vs_new"] = rel_l2(os.path.join(dumps, "old0"), os.path.join(dumps, "new0"))
    print("rel-L2 old vs new:", summary["rel_l2_old_vs_new"])
    if args.reps > 1:
        summary["rel_l2_old_vs_old"] = rel_l2(os.path.join(dumps, "old0"), os.path.join(dumps, "old1"))
        print("rel-L2 old vs old:", summary["rel_l2_old_vs_old"])
    shutil.rmtree(dumps, ignore_errors=True)
    if args.out:
        json.dump({"summary": summary, "runs": res}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
