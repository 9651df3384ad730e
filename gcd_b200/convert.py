"""Kubric-4D and ParDom-4D RGB-D scenes -> the merged point clouds `pcl_rgb_segm_*.pt` that evaluation reads (the reference's
"Dataset Processing" step: data-gen/convert_pcl_kubric.py, data-gen/convert_pcl_pardom.py).

Every pixel of every view of a frame is unprojected to world space and the views are stored together, one file per frame:
  Kubric  `pcl_rgb_segm_{t:05d}.pt`        = [xyz fp16 [16, H*W, 3], rgb u8 [16, H*W, 3], segm_rgb u8 [16, H*W, 3]], t < 60;
  ParDom  `pcl_rgb_segm_{10 t + 5:06d}.pt` = [xyz fp16 [19, H*W, 3], rgb u8 [19, H*W, 3], segm u8 [19, H*W, 1], tag u8 [19, H*W, 1]],
          t < 50, tag = view index; a frame with a missing file is skipped.
These are the files `evaluate.load_kubric_clouds` / `load_pardom_clouds` and the reference's data modules read.

The depth -> xyz arithmetic runs in one sm_90a kernel per frame (ops.unproject_depth, csrc/unproject.cu). The colour planes need no
arithmetic: the reference stores `uint8(float32(byte / 255) * 255)`, which is the byte itself for all 256 values, so they are the
decoded PNG bytes and never go to the device. The host reads the files as the reference does:
  * PNGs through PIL with matplotlib's `imread` rules: 8-bit RGB / RGBA as they are, palette (P) and grey + alpha (LA) converted to
    RGBA first. 16-bit PNGs (which matplotlib coarsens or scales differently) and greyscale PNGs (2-D arrays that the reference's
    `[..., 0:3]` / `[..., 0]` would slice along the columns) are refused with the file named.
  * Kubric depth TIFFs through PIL as float32; ParDom `npz['data']` as float32, which must hold H*W values.
  * Cameras as the reference builds them: pyquaternion's `Quaternion(q).rotation_matrix`, restated in float64 numpy below
    (normalised when not unit, as pyquaternion does), cast to float32; Kubric's extrinsic columns 1 and 2 negated and |K| scaled by
    the scene resolution. pyquaternion and matplotlib are not dependencies of this package, so neither is imported.

`convert_scene` decodes frames on a small thread pool, so that the next frames decode while the current one is on the device and the
previous one is written. Files are written under a temporary name that does not end in `.pt` and renamed, so a killed run never
leaves a truncated file that the skip rule (`ignore_if_exist`: a scene whose output holds at least 60 / 50 `*.pt` files is done)
would count. Scenes that fail are reported and the run goes on, as the reference's ParDom script does; the command then exits
non-zero and lists them.

    python -m gcd_b200.convert --kind kubric --input-root /datasets/Kubric-4D/data --output-root /datasets/Kubric-4D/pcl \\
        --examples eval/list/kubric_test20.txt

With --examples, each line's last path component names a scene under --input-root; without, the scenes are
`sorted(d for d in listdir(input_root) if 'scn' in d)[start_idx:end_idx]` ('scene' for ParDom). Under torchrun each rank takes
`pipeline.shard_clips` of the scenes.
"""
import argparse
import concurrent.futures as cf
import glob
import json
import os
import sys
import time

import numpy as np
import torch

KUBRIC_VIEWS, KUBRIC_FRAMES = 16, 60        # convert_pcl_kubric.py:282-283
PARDOM_VIEWS, PARDOM_FRAMES = 19, 50        # convert_pcl_pardom.py:269-270
PARDOM_MAX_DEPTH = 30000.0                  # convert_pcl_pardom.py:51: below half of fp16's largest value
DECODE_THREADS = 4
CAM = 16                                    # GCD_UNPROJECT_CAM: fx, fy, cx, cy, R (row-major), t

EXPECT_FILES = {"kubric": KUBRIC_FRAMES, "pardom": PARDOM_FRAMES}
SCENE_TAG = {"kubric": "scn", "pardom": "scene"}


# ---------------------------------------------------------------------------------------------------------------------------
# readers

_PNG_SIG = b"\x89PNG\r\n\x1a\n"
_PNG_COLOR = {0: "greyscale", 2: "RGB", 3: "palette", 4: "greyscale + alpha", 6: "RGBA"}


def read_png(path, channels):
    """uint8 [H, W, 3] (channels 0..2) or [H, W] (channel 0) of a PNG as matplotlib's imread(...) * 255 gives it back."""
    from PIL import Image
    with open(path, "rb") as f:
        head = f.read(26)
    if len(head) < 26 or head[:8] != _PNG_SIG or head[12:16] != b"IHDR":
        raise ValueError(f"{path}: not a PNG file")
    depth, color = head[24], head[25]
    if depth == 16:
        raise ValueError(f"{path}: 16-bit PNG ({_PNG_COLOR.get(color, color)}); only 8-bit PNGs are read as the reference reads them")
    if color == 0:
        raise ValueError(f"{path}: greyscale PNG; the reference slices channels of a [H, W, C] image, which a 2-D image does not have")
    if color not in _PNG_COLOR or (color != 3 and depth != 8):
        raise ValueError(f"{path}: unsupported PNG (bit depth {depth}, colour type {color})")
    with Image.open(path) as im:
        if im.mode in ("P", "LA"):
            im = im.convert("RGBA")
        if im.mode not in ("RGB", "RGBA"):
            raise ValueError(f"{path}: unexpected PIL mode {im.mode}")
        a = np.asarray(im)
    return np.ascontiguousarray(a[..., 0:3] if channels == 3 else a[..., 0])


def read_tiff_depth(path):
    """float32 [H, W] of a Kubric depth TIFF (np.array(PIL.Image.open(path)) cast to float32)."""
    from PIL import Image
    with Image.open(path) as im:
        a = np.array(im).astype(np.float32)
    if a.ndim != 2:
        raise ValueError(f"{path}: depth must be one channel, got shape {a.shape}")
    return a


def read_npz_depth(path, H, W):
    """float32 [H, W] of a ParDom depth file (np.load(path)['data'], which must hold H*W values)."""
    with np.load(path) as z:
        if "data" not in z:
            raise ValueError(f"{path}: no 'data' array")
        a = np.asarray(z["data"]).astype(np.float32)
    if a.size != H * W:
        raise ValueError(f"{path}: depth holds {a.size} values ({a.shape}), the frame has {H} x {W}")
    return a.reshape(H, W)


# ---------------------------------------------------------------------------------------------------------------------------
# cameras


def quaternion_rotation_matrix(q):
    """pyquaternion's `Quaternion(q).rotation_matrix` in float64 (q = w, x, y, z): normalised when |q|^2 is not within 1e-14 of 1,
    then the lower-right 3 x 3 of Q(q) Q_bar(q)^T."""
    q = np.array(q, dtype=np.float64).reshape(4)
    ss = np.dot(q, q)
    if not abs(1.0 - ss) < 1e-14:
        n = np.sqrt(ss)
        if n > 0:
            q = q / n
    w, x, y, z = q
    qm = np.array([[w, -x, -y, -z], [x, w, -z, y], [y, z, w, -x], [z, -y, x, w]])
    qb = np.array([[w, -x, -y, -z], [x, w, z, -y], [y, -z, w, x], [z, y, -x, w]])
    return np.dot(qm, qb.conj().transpose())[1:][:, 1:]


def _cam_row(K, RT):
    return np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2]], RT[0:3, 0:3].reshape(-1), RT[0:3, 3]]).astype(np.float32)


def kubric_cameras(scene_dir, num_frames=KUBRIC_FRAMES):
    """float32 [num_frames, 16 views, 16] camera rows of a Kubric scene (get_kubric_camera_matrices_torch, the |K| scaling by
    `scene.resolution` (W, H)), and the resolution (H, W)."""
    name = os.path.basename(os.path.normpath(scene_dir))
    cams = np.zeros((num_frames, KUBRIC_VIEWS, CAM), np.float32)
    hw = None
    for v in range(KUBRIC_VIEWS):
        path = os.path.join(scene_dir, f"{name}_p0_v{v}.json")
        with open(path) as f:
            meta = json.load(f)
        T = meta["scene"]["num_frames"]
        if T < num_frames:
            raise ValueError(f"{path}: {T} frames, the conversion needs {num_frames}")
        W, H = meta["scene"]["resolution"]
        if hw is None:
            hw = (int(H), int(W))
        K = np.abs(np.asarray(meta["camera"]["K"], dtype=np.float64)).astype(np.float32)
        if K.shape != (3, 3):
            raise ValueError(f"{path}: camera K must be 3 x 3, got {K.shape}")
        K[0, :] *= np.float32(W)
        K[1, :] *= np.float32(H)
        for t in range(num_frames):
            RT = np.eye(4, dtype=np.float32)
            RT[0:3, 0:3] = quaternion_rotation_matrix(meta["camera"]["quaternions"][t])
            RT[0:3, 3] = np.asarray(meta["camera"]["positions"][t], dtype=np.float64)
            RT[0:3, 1] *= -1.0
            RT[0:3, 2] *= -1.0
            cams[t, v] = _cam_row(K, RT)
    return cams, hw


def pardom_views(scene_dir):
    """The 19 views of a ParDom scene: the first 19 of sorted(listdir(<scene>/rgb)) (camera0, camera1, camera10, ..., yaw-0, ...)."""
    views = sorted(os.listdir(os.path.join(scene_dir, "rgb")))
    if len(views) < PARDOM_VIEWS:
        raise ValueError(f"{os.path.join(scene_dir, 'rgb')}: {len(views)} views, expected {PARDOM_VIEWS}")
    return views[:PARDOM_VIEWS]


def pardom_cameras(scene_dir, views):
    """float32 [V, 16] camera rows of a ParDom scene from its first calibration/*.json (constant over time)."""
    paths = glob.glob(os.path.join(scene_dir, "calibration", "*.json"))
    if not paths:
        raise FileNotFoundError(os.path.join(scene_dir, "calibration", "*.json"))
    with open(paths[0]) as f:
        cal = json.load(f)
    rows = {}
    for name, i, e in zip(cal["names"], cal["intrinsics"], cal["extrinsics"]):
        K = np.array([[i["fx"], 0.0, i["cx"]], [0.0, i["fy"], i["cy"]], [0.0, 0.0, 1.0]], dtype=np.float32)
        r, t = e["rotation"], e["translation"]
        RT = np.eye(4, dtype=np.float32)
        RT[0:3, 0:3] = quaternion_rotation_matrix([r["qw"], r["qx"], r["qy"], r["qz"]])
        RT[0:3, 3] = np.array([t["x"], t["y"], t["z"]], dtype=np.float32)
        rows[name] = _cam_row(K, RT)
    missing = [v for v in views if v not in rows]
    if missing:
        raise ValueError(f"{paths[0]}: no camera for views {missing}")
    return np.stack([rows[v] for v in views])


# ---------------------------------------------------------------------------------------------------------------------------
# frames


def kubric_frame_paths(scene_dir, t):
    return [(os.path.join(scene_dir, f"frames_p0_v{j}", f"rgba_{t:05d}.png"),
             os.path.join(scene_dir, f"frames_p0_v{j}", f"depth_{t:05d}.tiff"),
             os.path.join(scene_dir, f"frames_p0_v{j}", f"segmentation_{t:05d}.png")) for j in range(KUBRIC_VIEWS)]


def pardom_frame_paths(scene_dir, views, t):
    s = f"{t * 10 + 5:018d}"
    return [(os.path.join(scene_dir, "rgb", v, s + ".png"), os.path.join(scene_dir, "depth", v, s + ".npz"),
             os.path.join(scene_dir, "semantic_segmentation_2d", v, s + ".png")) for v in views]


def output_name(kind, t):
    return f"pcl_rgb_segm_{t:05d}.pt" if kind == "kubric" else f"pcl_rgb_segm_{t * 10 + 5:06d}.pt"


def decode_frame(kind, paths):
    """Reads one frame of all views. Returns (depth float32 [V, H, W], rgb u8 [V, N, 3], segm u8 [V, N, 3] (Kubric) or [V, N, 1]
    (ParDom)), or None for a ParDom frame with a missing file."""
    if kind == "pardom" and not all(os.path.isfile(p) for trio in paths for p in trio):
        return None
    depth, rgb, segm = [], [], []
    for rgb_p, depth_p, segm_p in paths:
        c = read_png(rgb_p, 3)
        H, W = c.shape[:2]
        if kind == "kubric":
            d = read_tiff_depth(depth_p)
            s = read_png(segm_p, 3)
        else:
            d = read_npz_depth(depth_p, H, W)
            s = read_png(segm_p, 1)[..., None]
        for p, a in ((depth_p, d), (segm_p, s)):
            if a.shape[:2] != (H, W):
                raise ValueError(f"{p}: {a.shape[0]} x {a.shape[1]} pixels, {rgb_p} has {H} x {W}")
        if rgb and c.shape != rgb[0].shape:
            raise ValueError(f"{rgb_p}: {H} x {W} pixels, the frame's first view has {rgb[0].shape[0]} x {rgb[0].shape[1]}")
        depth.append(d)
        rgb.append(c)
        segm.append(s)
    V, (H, W) = len(paths), rgb[0].shape[:2]
    return np.stack(depth), np.stack(rgb).reshape(V, H * W, 3), np.stack(segm).reshape(V, H * W, -1)


def save_frame(path, tensors):
    """torch.save(tensors) to `path` through a temporary name that does not end in .pt, then an atomic rename."""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        torch.save(tensors, f)
    os.replace(tmp, path)


def is_finished(out_dir, kind):
    """The reference's skip rule: at least 60 (Kubric) / 50 (ParDom) `*.pt` files in the scene's output directory."""
    return len(glob.glob(os.path.join(out_dir, "*.pt"))) >= EXPECT_FILES[kind]


class _Device:
    """Upload, kernel and download of one frame; the fp16 result lands in a pinned host buffer."""

    def __init__(self, kind, device):
        self.mode = 1 if kind == "kubric" else 0                   # ops.UNPROJECT_BALL_TO_PLANE / UNPROJECT_CLAMP
        self.max_depth = 0.0 if kind == "kubric" else PARDOM_MAX_DEPTH
        self.device = torch.device(device)
        self.shape = None
        self.uploaded = None

    def _alloc(self, V, H, W):
        if self.shape != (V, H, W):
            self.depth_h = torch.empty((V, H, W), dtype=torch.float32).pin_memory()
            self.depth_d = torch.empty((V, H, W), dtype=torch.float32, device=self.device)
            self.xyz_d = torch.empty((V, H * W, 3), dtype=torch.float16, device=self.device)
            self.shape = (V, H, W)

    def upload(self, depth, cams_d):
        V, H, W = depth.shape
        self._alloc(V, H, W)
        if self.uploaded is not None:
            self.uploaded.synchronize()         # the previous frame's copy has left the pinned buffer
        self.cams_d = cams_d
        self.depth_h.numpy()[...] = depth
        self.depth_d.copy_(self.depth_h, non_blocking=True)
        self.uploaded = torch.cuda.Event()
        self.uploaded.record()

    def kernel(self):
        from . import ops
        ops.unproject_depth(self.depth_d, self.cams_d, self.mode, self.xyz_d, self.max_depth)

    def download(self):
        """Copies xyz into a fresh pinned tensor; returns it with an event that completes with the copy."""
        out = torch.empty(self.xyz_d.shape, dtype=torch.float16).pin_memory()
        out.copy_(self.xyz_d, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return out, ev


def _frames_of(kind, scene_dir):
    """[(t, per-view paths)], camera rows per frame (numpy [T, V, 16] or [V, 16])."""
    if kind == "kubric":
        cams, _ = kubric_cameras(scene_dir)
        return [(t, kubric_frame_paths(scene_dir, t)) for t in range(KUBRIC_FRAMES)], cams
    views = pardom_views(scene_dir)
    cams = pardom_cameras(scene_dir, views)
    return [(t, pardom_frame_paths(scene_dir, views, t)) for t in range(PARDOM_FRAMES)], cams


def _save_job(path, xyz, ev, rgb, segm, kind, V):
    ev.synchronize()
    lst = [xyz.clone(), torch.from_numpy(rgb), torch.from_numpy(segm)]
    if kind == "pardom":
        lst.append(torch.arange(V, dtype=torch.uint8)[:, None, None].expand(V, rgb.shape[1], 1).contiguous())
    save_frame(path, lst)


def convert_scene(kind, scene_dir, out_dir, device="cuda"):
    """Converts one scene. Returns {"frames": written, "skipped_frames": [t of ParDom frames with a missing file]}."""
    if kind not in EXPECT_FILES:
        raise ValueError(f"kind must be kubric or pardom, got {kind!r}")
    frames, cams = _frames_of(kind, scene_dir)
    dev = _Device(kind, device)
    cams_d = torch.from_numpy(cams).to(dev.device)
    os.makedirs(out_dir, exist_ok=True)
    written, skipped = 0, []
    with cf.ThreadPoolExecutor(DECODE_THREADS) as dec, cf.ThreadPoolExecutor(1) as sav:
        pending = [dec.submit(decode_frame, kind, p) for _, p in frames[:DECODE_THREADS]]
        saves = []
        for i, (t, _) in enumerate(frames):
            got = pending[i].result()
            if i + DECODE_THREADS < len(frames):
                pending.append(dec.submit(decode_frame, kind, frames[i + DECODE_THREADS][1]))
            pending[i] = None
            if got is None:
                skipped.append(t)
                continue
            depth, rgb, segm = got
            dev.upload(depth, cams_d[t] if kind == "kubric" else cams_d)
            dev.kernel()
            xyz, ev = dev.download()
            saves = [s for s in saves if not s.done() or s.result()]
            if len(saves) >= 2:                 # at most two frames wait to be written
                saves.pop(0).result()
            saves.append(sav.submit(_save_job, os.path.join(out_dir, output_name(kind, t)), xyz, ev, rgb, segm, kind,
                                    depth.shape[0]))
            written += 1
        for s in saves:
            s.result()
    return {"frames": written, "skipped_frames": skipped}


# ---------------------------------------------------------------------------------------------------------------------------
# command line


def discover_scenes(kind, input_root, examples=None, start_idx=0, end_idx=None):
    """Scene directory names: the last path component of each line of `examples` (evaluate.read_examples), or the reference's
    `sorted(d for d in listdir(input_root) if tag in d)[start_idx:end_idx]`."""
    if examples:
        from .evaluate import read_examples
        return [os.path.basename(os.path.normpath(e)) for e in read_examples(examples)]
    names = sorted(d for d in os.listdir(input_root) if SCENE_TAG[kind] in d)
    return names[start_idx:end_idx]


def parser():
    p = argparse.ArgumentParser(prog="python -m gcd_b200.convert",
                                description="Convert Kubric-4D / ParDom-4D RGB-D scenes to the merged point clouds evaluation reads.")
    p.add_argument("--kind", choices=["kubric", "pardom"], required=True)
    p.add_argument("--input-root", required=True, help="directory holding the scene directories")
    p.add_argument("--output-root", required=True, help="<output-root>/<scene>/pcl_rgb_segm_*.pt is written")
    p.add_argument("--examples", default="", help="text file with one scene per line (eval/list/*_test*.txt); its last path "
                                                  "component names the scene under --input-root")
    p.add_argument("--start-idx", type=int, default=None)
    p.add_argument("--end-idx", type=int, default=None)
    p.add_argument("--overwrite", action="store_true", help="convert scenes the skip rule would consider finished")
    return p


def main(argv=None):
    from .pipeline import shard_clips
    args = parser().parse_args(argv)
    if args.examples and (args.start_idx is not None or args.end_idx is not None):
        raise SystemExit("--examples and --start-idx / --end-idx exclude each other")
    if not os.path.isdir(args.input_root):
        raise SystemExit(f"--input-root {args.input_root} is not a directory")
    if args.examples and not os.path.isfile(args.examples):
        raise SystemExit(f"--examples {args.examples} is not a file")
    if not torch.cuda.is_available():
        raise SystemExit("gcd_b200.convert runs on a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = f"cuda:{int(os.environ.get('LOCAL_RANK', 0))}"
    torch.cuda.set_device(device)
    names = discover_scenes(args.kind, args.input_root, args.examples, args.start_idx or 0, args.end_idx)
    failed = []
    for i in shard_clips(len(names), rank, world):
        name = names[i]
        scene, out = os.path.join(args.input_root, name), os.path.join(args.output_root, name)
        rec = {"scene": name, "index": i, "output": out}
        if not args.overwrite and is_finished(out, args.kind):
            rec["status"] = "skipped"
        else:
            t0 = time.perf_counter()
            try:
                rec.update(convert_scene(args.kind, scene, out, device))
                rec["status"] = "done"
            except Exception as e:      # reported, and the run goes on (convert_pcl_pardom.py:252-257)
                rec.update(status="failed", error=f"{type(e).__name__}: {e}")
                failed.append(name)
            rec["seconds"] = round(time.perf_counter() - t0, 3)
        print(json.dumps(rec), flush=True)
    if failed:
        print(f"gcd_b200.convert: {len(failed)} scene(s) failed: {' '.join(failed)}", file=sys.stderr, flush=True)
        raise SystemExit(1)
    return 0


if __name__ == "__main__":
    main()
