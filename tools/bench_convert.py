"""Times gcd_b200.convert on one seeded full-size Kubric scene (16 views of 384 x 576) and one ParDom scene (19 views of 480 x 640),
written to a temporary directory with --frames frames each.

    python tools/bench_convert.py [--frames 8] [--reps 3] [--out results.json]

Per frame, stage by stage in a serial loop with a device synchronise after each stage (host clock): decode (PNG / TIFF / npz reads),
upload (depth into pinned memory and to the device), kernel (gcd_unproject_depth), download (xyz into pinned memory), save
(torch.save + rename). Frames/s of `convert_scene` (decode pool, device and writer overlapped) against that serial loop, and against
the oracle's per-view float32 torch chain on the same GPU (oracle/pcl_oracle.torch_chain: the reference's device work; its host
reads go through matplotlib, which this package does not install, so the chain is timed from decoded depth). The kernel alone:
CUDA events over 50 launches on device-resident depth, GB/s of its 10 bytes per pixel against the 3.35 TB/s data-sheet bound.
Best of --reps; the card name and power limit are read in the same run."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import convert as C, ops  # noqa: E402
from oracle import pcl_oracle as P  # noqa: E402
from tools.bench_lpips import card  # noqa: E402

HBM = 3.35e12


def _sync_time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def serial(kind, scene, out_dir, frames):
    """The stages one after another; returns per-stage seconds per frame and the total."""
    fr, cams = C._frames_of(kind, scene)
    fr = [x for x in fr if x[0] < frames]
    dev = C._Device(kind, "cuda")
    cams_d = torch.from_numpy(cams).cuda()
    st = dict(decode=0.0, upload=0.0, kernel=0.0, download=0.0, save=0.0)
    os.makedirs(out_dir, exist_ok=True)
    for t, paths in fr:
        dt, got = _sync_time(lambda: C.decode_frame(kind, paths))
        st["decode"] += dt
        depth, rgb, segm = got
        st["upload"] += _sync_time(lambda: dev.upload(depth, cams_d[t] if kind == "kubric" else cams_d))[0]
        st["kernel"] += _sync_time(dev.kernel)[0]
        dt, (xyz, ev) = _sync_time(dev.download)
        st["download"] += dt
        st["save"] += _sync_time(lambda: C._save_job(os.path.join(out_dir, C.output_name(kind, t)), xyz, ev, rgb, segm, kind,
                                                     depth.shape[0]))[0]
    n = len(fr)
    return {k: v / n * 1e3 for k, v in st.items()}, sum(st.values()) / n


def torch_chain_time(kind, depth, cams):
    dt, _ = _sync_time(lambda: P.torch_chain(depth, cams, kind, "cuda").cpu())
    return dt


def kernel_alone(kind, depth, cams):
    d = torch.from_numpy(depth).cuda()
    c = torch.from_numpy(cams).cuda()
    out = torch.empty((d.shape[0], d.shape[1] * d.shape[2], 3), dtype=torch.float16, device="cuda")
    mode = ops.UNPROJECT_BALL_TO_PLANE if kind == "kubric" else ops.UNPROJECT_CLAMP
    for _ in range(5):
        ops.unproject_depth(d, c, mode, out, C.PARDOM_MAX_DEPTH)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        ops.unproject_depth(d, c, mode, out, C.PARDOM_MAX_DEPTH)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 50
    by = d.numel() * 10
    return ms, by / (ms * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_convert needs a CUDA device"
    res = {"card": card(), "frames": a.frames}
    tmp = tempfile.mkdtemp()
    try:
        for kind, hw in (("kubric", (384, 576)), ("pardom", (480, 640))):
            H, W = hw
            t0 = time.perf_counter()
            if kind == "kubric":
                scene = P.write_kubric_scene(os.path.join(tmp, "data"), "scn00001", H, W, C.KUBRIC_FRAMES, 1)
            else:
                scene = P.write_pardom_scene(os.path.join(tmp, "data"), "scene_000001", H, W, C.PARDOM_FRAMES, 2)
            write_s = time.perf_counter() - t0
            out = os.path.join(tmp, "pcl")
            frames = C.KUBRIC_FRAMES if kind == "kubric" else C.PARDOM_FRAMES
            stages, ser, full, chain = None, [], [], []
            depth, _, _ = C.decode_frame(kind, C._frames_of(kind, scene)[0][0][1])
            cams = C._frames_of(kind, scene)[1]
            cams0 = cams[0] if kind == "kubric" else cams
            torch_chain_time(kind, depth, cams0)                      # warm-up
            for _ in range(a.reps):
                shutil.rmtree(out, ignore_errors=True)
                s, tot = serial(kind, scene, os.path.join(out, "serial"), a.frames)
                stages = s if stages is None or tot * 1e3 < sum(stages.values()) else stages
                ser.append(tot)
                shutil.rmtree(out, ignore_errors=True)
                dt, _ = _sync_time(lambda: C.convert_scene(kind, scene, os.path.join(out, "full"), "cuda"))
                full.append(dt / frames)
                chain.append(torch_chain_time(kind, depth, cams0))
            ms, gbs = kernel_alone(kind, depth, cams0)
            r = dict(views=int(depth.shape[0]), hw=hw, scene_write_s=round(write_s, 1),
                     stage_ms_per_frame={k: round(v, 3) for k, v in stages.items()},
                     serial_frames_per_s=round(1 / min(ser), 2), convert_scene_frames_per_s=round(1 / min(full), 2),
                     torch_chain_device_ms_per_frame=round(min(chain) * 1e3, 3), kernel_ms=round(ms, 4), kernel_gb_s=round(gbs, 1),
                     kernel_share_of_hbm_bound=round(gbs * 1e9 / HBM, 3))
            res[kind] = r
            print(json.dumps({kind: r}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
