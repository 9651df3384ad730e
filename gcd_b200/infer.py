"""GCD on arbitrary input videos and images, on the device: the path of gcd-model/scripts/infer.py from an mp4, a folder of frames
or a single image to the predicted videos and their per-pixel uncertainty across samples.

    inputs (list_inputs) -> decoded uint8 frames (read_frames) -> crop + resize on the device (prepare_frames: gcd_frames_prepare)
    -> batch (construct_batch) -> evaluate.sample_example -> metrics.sample_diversity -> frame folders / mp4 (save_results)

Input discovery, the crop box, frame selection, the batch and the output names restate the reference's host code
(eval_utils.py, sgm/data/common.py, infer.py) operation for operation. The per-pixel work (u8 / 255, centre crop,
cv2 INTER_LINEAR resize, the `* 2 - 1` / `(x + 1) / 2` round trip) is one kernel launch per group of equally sized frames.

Command line (one result set per example under <output>/extra/; under torchrun each rank takes `pipeline.shard_clips`):

    python -m gcd_b200.infer --kind kubric --checkpoint kubric_gradual_max90.ckpt --input my_clip.mp4 --output out/demo_run \\
        --delta-azimuth 30 --delta-elevation 15 --max-delta-azimuth 90 --max-delta-elevation 30
"""
import argparse
import glob
import json
import os
import sys

import numpy as np
import torch

from . import evaluate

IMAGE_EXTENSIONS = (".jpg", ".jpeg", ".png", ".bmp", ".tiff")          # sgm/data/common.py:22-23
VIDEO_EXTENSIONS = (".mp4", ".avi", ".mov", ".flv", ".mkv", ".webm")
TRAINED_HW = (256, 384)                                                # every shipped GCD checkpoint


# ---------------------------------------------------------------------------------------------------------------------------
# input discovery (eval_utils.py:311-413)


def is_image_file(path):
    return os.path.splitext(path)[1].lower() in IMAGE_EXTENSIONS


def is_video_file(path):
    return os.path.splitext(path)[1].lower() in VIDEO_EXTENSIONS


def is_image_folder(path):
    """True when more than half of the directory's entries are image files (eval_utils.is_image_folder: its
    `(count > n / 2) > 0.8` compares a bool with 0.8, which is this)."""
    entries = os.listdir(path)
    images = sum(1 for f in entries if os.path.isfile(os.path.join(path, f)) and is_image_file(f))
    return images > len(entries) / 2


def list_inputs(paths):
    """The examples named by `paths` (eval_utils.get_list_of_input_images_or_videos): a path that does not exist is a glob; an
    image or video file is an example; a `.txt` file lists examples one per line (blank lines and lines starting with `#`
    skipped; the lines are taken as they are); an image folder is an example; any other directory is searched, sorted, through
    its subdirectories."""
    out = []
    for path in paths:
        if not os.path.exists(path):
            out.extend(glob.glob(path))
        elif os.path.isfile(path):
            if is_image_file(path) or is_video_file(path):
                out.append(path)
            if path.lower().endswith(".txt"):
                with open(path) as f:
                    lines = [ln.strip() for ln in f.readlines()]
                out.extend(ln for ln in lines if ln and not ln.startswith("#"))
        elif os.path.isdir(path):
            if is_image_folder(path):
                out.append(path)
            else:
                subs = [os.path.join(path, f) for f in sorted(os.listdir(path))]
                out.extend(list_inputs([d for d in subs if os.path.isdir(d)]))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# readers: uint8 frames, cropped and resized on the device


def crop_box(H, W, frame_hw, center_crop=True):
    """(y0, x0, ch, cw) of center_crop_numpy(image, frame_width / frame_height) on an H x W frame (common.py:87-118): the width is
    cropped to int(H * ar) when W / H exceeds the target aspect by more than 2e-3, the height to int(W / ar) when it falls short
    by more than 2e-3, offsets (H - ch) // 2 and (W - cw) // 2. center_crop False keeps the whole frame."""
    fh, fw = frame_hw
    if not center_crop:
        return 0, 0, H, W
    ar = fw / fh
    video_ar = W / H
    if video_ar > ar + 2e-3:
        ch, cw = H, int(H * ar)
    elif video_ar < ar - 2e-3:
        ch, cw = int(W / ar), W
    else:
        return 0, 0, H, W
    return (H - ch) // 2, (W - cw) // 2, ch, cw


def clip_frames(num_frames, frame_start, frame_stride):
    """Frame indices of the clip (infer.py:127-132)."""
    if frame_start < 0 or frame_stride < 0:
        raise ValueError(f"frame_start {frame_start} and frame_stride {frame_stride} must be >= 0")
    return np.arange(num_frames) * int(frame_stride) + int(frame_start)


def _check_u8(img, path):
    if img.dtype != torch.uint8:
        raise ValueError(f"{path}: {img.dtype} image; only 8-bit images are read")
    if img.shape[0] not in (3, 4):
        raise ValueError(f"{path}: {img.shape[0]}-channel image; only RGB / RGBA images are read (grayscale is not)")
    return img.permute(1, 2, 0).contiguous()


def read_image(path):
    """uint8 [H, W, 3 | 4] of an 8-bit RGB / RGBA image file (torchvision.io)."""
    from torchvision.io import ImageReadMode, decode_image, read_file
    return _check_u8(decode_image(read_file(path), mode=ImageReadMode.UNCHANGED), path)


def read_video(path, frames):
    """uint8 BGR [len(frames), H, W, 3] of the given frames of a video file, decoded with cv2.VideoCapture up to the last of
    them."""
    try:
        import cv2
    except ImportError:
        raise ImportError(f"{path}: reading video files needs OpenCV (cv2)") from None
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        raise ValueError(f"{path}: cannot open the video")
    want, last, got = set(int(t) for t in frames), int(max(frames)), {}
    try:
        for t in range(last + 1):
            ok, img = cap.read()
            if not ok:
                raise ValueError(f"{path}: clip frames {int(min(frames))}..{last} run past the {t} frames of the video")
            if t in want:
                if img.ndim != 3 or img.dtype != np.uint8 or img.shape[2] != 3:
                    raise ValueError(f"{path}: decoded {img.dtype} frames of shape {img.shape}; only 8-bit colour video is read")
                got[t] = torch.from_numpy(img)
    finally:
        cap.release()
    return torch.stack([got[int(t)] for t in frames])


def read_frames(example, frames):
    """Decoded frames of an example: (list of uint8 [H, W, C] tensors, one per clip frame, channel map). Frames of a single
    image are the same tensor (a still); a video's are BGR (channel map (2, 1, 0)), the others RGB."""
    frames = [int(t) for t in frames]
    if is_image_file(example):
        img = read_image(example)
        return [img] * len(frames), (0, 1, 2)
    if os.path.isfile(example):
        return list(read_video(example, frames)), (2, 1, 0)
    if not os.path.isdir(example):
        raise ValueError(f"invalid input path: {example}")
    if "kubgen" in example:                                   # common.load_kubric_video_rgb_frames
        paths = [os.path.join(example, f"rgba_{t:05d}.png") for t in frames]
    else:                                                     # common.load_video_all_frames
        found = [p for p in sorted(glob.glob(os.path.join(example, "*.*"))) if is_image_file(p)]
        if frames[-1] >= len(found):
            raise ValueError(f"{example}: clip frames {frames[0]}..{frames[-1]} run past its {len(found)} images")
        paths = [found[t] for t in frames]
    return [read_image(p) for p in paths], (0, 1, 2)


def prepare_frames(images, frame_hw, center_crop=True, channel_map=(0, 1, 2), device="cuda"):
    """infer.py's input_rgb: float32 [len(images), 3, h, w] in [0, 1] on `device` from uint8 [H, W, 3 | 4] frames (any mix of
    sizes): per frame the centre crop of crop_box, cv2 INTER_LINEAR to frame_hw and the fp32 round trip `((p * 2 - 1) + 1) / 2`,
    in one gcd_frames_prepare launch per group of equally shaped frames. Repeated tensors (a still) are prepared once."""
    from . import ops
    out = torch.empty(len(images), 3, *frame_hw, device=device, dtype=torch.float32)
    groups, first = {}, {}
    for i, img in enumerate(images):
        if id(img) in first:
            continue
        first[id(img)] = i
        groups.setdefault(tuple(img.shape), []).append(i)
    for shape, idx in groups.items():
        frames = torch.stack([images[i] for i in idx]).to(device)
        box = crop_box(shape[0], shape[1], frame_hw, center_crop)
        dest = torch.tensor(idx, dtype=torch.int32).to(device)
        ops.frames_prepare(frames, box, out, channel_map, dest)
    for i, img in enumerate(images):
        if first[id(img)] != i:
            out[i] = out[first[id(img)]]
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# batch (eval_utils.py:191-263)


def camera_control(kind):
    """The conditioning the shipped configs train with: Kubric spherical angles, ParDom none."""
    return "spherical" if kind == "kubric" else "none"


def construct_batch(kind, input_rgb, delta_azimuth, delta_elevation, delta_radius, frame_rate, motion_id, cond_aug, generator,
                    force_custom_mbid=False, trajectory="interpol_linear", move_time=13, delta_azimuth_range=(-180.0, 180.0),
                    delta_elevation_range=(-60.0, 60.0), motion_bucket_range=None):
    """The model batch of a custom clip (eval_utils.construct_batch for infer.py).

    input_rgb: [T, 3, H, W] in [0, 1] (prepare_frames) on any device; the frames become `* 2 - 1` on that device. frame_rate,
    delta_*: the command line's values, taken through float32 as infer.py's `controls` array does (so fps_id is float32, as
    the reference's); generator: the conditioning noise (cond_frames = x + randn * cond_aug) is drawn from it, on its own device.
    Kubric (spherical camera control): scaled_relative_angles [T, 3] of the trajectory from (0, 0, 0) to (Δaz, Δel, Δr) with
    azimuth / elevation in radians, and the motion bucket synchronised with the angular distance over the configured maximum
    unless force_custom_mbid or the bucket range is empty. ParDom (no camera control): motion_id as given, no angles.
    motion_bucket_range: default (0, 255) for Kubric, (127, 127) for ParDom."""
    if kind not in ("kubric", "pardom"):
        raise ValueError(f"unknown dataset kind {kind!r}")
    controls = np.array([0, 0, frame_rate, delta_azimuth, delta_elevation, delta_radius], dtype=np.float32)
    azimuth_deg, elevation_deg, radius_m, frame_rate = controls[3], controls[4], controls[5], controls[2]
    if motion_bucket_range is None:
        motion_bucket_range = (0, 255) if kind == "kubric" else (127, 127)
    control = camera_control(kind)
    T = input_rgb.shape[0]
    x = input_rgb.to(torch.float32) * 2.0 - 1.0
    noise = torch.randn(*x.shape, generator=generator, device=generator.device).to(x.device)
    batch = dict(motion_bucket_id=torch.ones(T, dtype=torch.int32) * motion_id,
                 fps_id=torch.ones(T, dtype=torch.int32) * frame_rate,
                 cond_aug=torch.ones(T, dtype=torch.float32) * cond_aug,
                 cond_frames_without_noise=x, cond_frames=x + noise * cond_aug, jpg=torch.zeros_like(x),
                 image_only_indicator=torch.zeros(1, T, dtype=torch.float32), num_video_frames=T)
    if control == "spherical":
        if not (np.isfinite(azimuth_deg) and np.isfinite(elevation_deg) and np.isfinite(radius_m)):
            raise ValueError("delta azimuth, elevation and radius must be finite")
        evaluate._check_move_time(move_time, T)
        start = np.array([0.0, 0.0, 0.0], dtype=np.float32)
        end = np.array([azimuth_deg, elevation_deg, radius_m], dtype=np.float32)
        src = np.tile(start[None], (T, 1))
        dst = np.tile(end[None], (T, 1))
        for t in range(move_time):                             # common.construct_trajectory
            a = evaluate._alpha(trajectory, t, move_time)
            dst[t] = start * (1.0 - a) + end * a
        angles = dst - src
        angles[:, 0] *= np.pi / 180.0
        angles[:, 1] *= np.pi / 180.0
        batch["scaled_relative_angles"] = torch.tensor(angles, dtype=torch.float32)
    lo, hi = motion_bucket_range
    if control != "none" and not force_custom_mbid and hi - lo > 0:
        motion = np.linalg.norm(end[0:2] - start[0:2], ord=2)
        motion_max = np.linalg.norm([max(*delta_azimuth_range), max(*delta_elevation_range)], ord=2)
        batch["motion_bucket_id"] = torch.ones(T, dtype=torch.int32) * int(round(lo + (hi - lo) * (motion / motion_max)))
    return batch


# ---------------------------------------------------------------------------------------------------------------------------
# outputs (infer.py:417-452, 499-522; eval_utils.write_video_and_frames)


def model_name(checkpoint):
    """infer.py's short model name (eval_utils.load_model_bundle): the run name of a training checkpoint, else the file name
    with kubric -> kb, pardom -> pd, gradual -> gr, direct -> di, semantic -> sem, max -> m."""
    if "/checkpoints" in checkpoint:
        return checkpoint.split("/checkpoints")[0].rsplit("_", 1)[-1]
    name = os.path.basename(checkpoint).split(".")[0]
    for k, v in (("kubric", "kb"), ("pardom", "pd"), ("gradual", "gr"), ("direct", "di"), ("semantic", "sem"), ("max", "m")):
        name = name.replace(k, v)
    return name


def output_stem(output, index, example, model):
    """<output>/extra/<tag>_<index:03d>_n<model>_<name>: tag is the output directory's name up to its first `_`, name the
    example's file or folder name without extension, `_p0` and `_rgb`."""
    tag = os.path.basename(output).split("_")[0]
    name = os.path.splitext(os.path.basename(example))[0].replace("_p0", "").replace("_rgb", "")
    return os.path.join(output, "extra", f"{tag}_{index:03d}_n{model}_{name}")


def quantize(x):
    """uint8(x * 255) by truncation, as eval_utils.write_video_and_frames (:524)."""
    return (x.to(torch.float32) * 255.0).to(torch.uint8)


def write_frames(frames, stem, fps, save_images, save_mp4):
    """frames: uint8 [T, C, H, W] (C = 3 RGB or 1 grayscale). Frame folder <stem>/0000.png ... and / or <stem>.mp4."""
    frames = frames.cpu()
    if save_images:
        from torchvision.io import write_png
        os.makedirs(stem, exist_ok=True)
        for i, f in enumerate(frames):
            write_png(f, os.path.join(stem, f"{i:04d}.png"))
    if save_mp4:
        import cv2
        os.makedirs(os.path.dirname(stem), exist_ok=True)
        T, C, H, W = frames.shape
        w = cv2.VideoWriter(stem + ".mp4", cv2.VideoWriter_fourcc(*"mp4v"), float(fps), (W, H))
        if not w.isOpened():
            raise RuntimeError(f"{stem}.mp4: cv2.VideoWriter cannot write mp4v video")
        for f in frames:
            img = f.permute(1, 2, 0).numpy()
            w.write(np.ascontiguousarray(np.repeat(img, 3, axis=2) if C == 1 else img[..., ::-1]))
        w.release()


def save_results(stem, input_rgb, sampled, uncertainty, diversity, fps, save_images=True, save_mp4=True, save_input=True,
                 save_uncertainty=True):
    """infer.py's save_results for the per-clip outputs: <stem>_input, <stem>_pred_s<s>, <stem>_uncert (clip(3 u, 0, 1) in
    grayscale: the reference's magma colouring is not reproduced), each a frame folder and / or an mp4, plus <stem>_metrics.json
    with frame_diversity / mean_diversity. input_rgb [T, 3, H, W], sampled [S, T, 3, H, W] in [0, 1]; uncertainty [T, H, W]."""
    frame_div, mean_div = diversity
    if save_images or save_mp4:
        if save_input:
            write_frames(quantize(input_rgb), stem + "_input", fps, save_images, save_mp4)
        for s in range(sampled.shape[0]):
            write_frames(quantize(sampled[s]), stem + f"_pred_s{s}", fps, save_images, save_mp4)
        if save_uncertainty:
            write_frames(quantize(torch.clamp(uncertainty * 3.0, 0.0, 1.0))[:, None], stem + "_uncert", fps, save_images, save_mp4)
    evaluate.save_metrics_json(stem + "_metrics.json", {"frame_diversity": frame_div, "mean_diversity": mean_div})


# ---------------------------------------------------------------------------------------------------------------------------
# command line


def _multiple_of_64(s):
    v = int(s)
    if v <= 0 or v % 64:
        raise argparse.ArgumentTypeError(f"{v} is not a positive multiple of 64 (the UNet halves the latent three times)")
    return v


def parser():
    p = argparse.ArgumentParser(prog="python -m gcd_b200.infer",
                                description="Run a GCD checkpoint on your own videos, frame folders or images (infer.py).")
    p.add_argument("--kind", choices=["kubric", "pardom"], required=True, help="the checkpoint's dataset: sets the conditioning")
    p.add_argument("--checkpoint", required=True, help=".ckpt or .safetensors with the DiffusionEngine's keys")
    p.add_argument("--use-ema", type=int, default=0)
    p.add_argument("--model-config", default="", help="JSON with unet / vae / encoder / vit overrides of the GCD shapes")
    p.add_argument("--input", nargs="+", required=True,
                   help="video files, image files, frame folders, directories of those, .txt lists or globs")
    p.add_argument("--output", required=True)
    p.add_argument("--num-samples", type=int, default=2)
    p.add_argument("--num-frames", type=int, default=14)
    p.add_argument("--num-steps", type=int, default=25)
    p.add_argument("--guider-max-scale", type=float, default=1.5)
    p.add_argument("--guider-min-scale", type=float, default=1.0)
    p.add_argument("--motion-id", type=int, default=127, help="motion bucket (Kubric models override it from the angles)")
    p.add_argument("--force-custom-mbid", type=int, default=0, help="1: keep --motion-id for Kubric models too")
    p.add_argument("--cond-aug", type=float, default=0.02)
    p.add_argument("--decoding-t", type=int, default=14)
    p.add_argument("--delta-azimuth", type=float, default=30.0)
    p.add_argument("--delta-elevation", type=float, default=15.0)
    p.add_argument("--delta-radius", type=float, default=0.0)
    p.add_argument("--frame-start", type=int, default=0)
    p.add_argument("--frame-stride", type=int, default=2)
    p.add_argument("--frame-rate", type=int, default=12)
    p.add_argument("--frame-width", type=_multiple_of_64, default=384)
    p.add_argument("--frame-height", type=_multiple_of_64, default=256)
    p.add_argument("--center-crop", type=int, default=1)
    p.add_argument("--save-images", type=int, default=1)
    p.add_argument("--save-mp4", type=int, default=1)
    p.add_argument("--save-input", type=int, default=1)
    p.add_argument("--save-uncertainty", type=int, default=1)
    p.add_argument("--seed", type=int, default=0, help="seeds the device generator of the conditioning and latent noise")
    p.add_argument("--trajectory", choices=["interpol_linear", "interpol_sine"], default="interpol_linear")
    p.add_argument("--move-time", type=int, default=13, help="frames the target camera moves over (gradual 13, direct 0)")
    p.add_argument("--max-delta-azimuth", type=float, default=180.0, help="Kubric motion normalisation (max-90 configs: 90)")
    p.add_argument("--max-delta-elevation", type=float, default=60.0, help="Kubric motion normalisation (max-90 configs: 30)")
    p.add_argument("--motion-bucket-range", type=int, nargs=2, default=None)
    return p


def warn_resolution_mismatch(frame_hw):
    if tuple(frame_hw) != TRAINED_HW:
        print(f"warning: the GCD checkpoints were trained at {TRAINED_HW[1]} x {TRAINED_HW[0]}, running inference at "
              f"{frame_hw[1]} x {frame_hw[0]}", file=sys.stderr, flush=True)


def prepare_input(args, example, generator, device):
    """(input_rgb [T, 3, h, w] in [0, 1] on the device, batch) of one example (infer.py load_input)."""
    hw = (args.frame_height, args.frame_width)
    images, cmap = read_frames(example, clip_frames(args.num_frames, args.frame_start, args.frame_stride))
    input_rgb = prepare_frames(images, hw, bool(args.center_crop), cmap, device)
    batch = construct_batch(args.kind, input_rgb, args.delta_azimuth, args.delta_elevation, args.delta_radius, args.frame_rate,
                            args.motion_id, args.cond_aug, generator, bool(args.force_custom_mbid), args.trajectory,
                            args.move_time, (-args.max_delta_azimuth, args.max_delta_azimuth),
                            (-args.max_delta_elevation, args.max_delta_elevation), args.motion_bucket_range)
    return input_rgb, batch


def example_generator(seed, index, device):
    return torch.Generator(device=device).manual_seed(seed * 1000003 + index)


def main(argv=None):
    from . import metrics
    from .pipeline import shard_clips
    args = parser().parse_args(argv)
    if args.save_mp4:
        try:
            import cv2  # noqa: F401
        except ImportError:
            raise SystemExit("--save-mp4 1 needs OpenCV (cv2) to write the videos; install it or pass --save-mp4 0")
    if args.num_samples < 1:
        raise SystemExit("--num-samples must be >= 1")
    examples = list_inputs(args.input)
    if not examples:
        raise SystemExit(f"no videos, images or frame folders found in {args.input}")
    if not torch.cuda.is_available():
        raise SystemExit("gcd_b200.infer runs on a CUDA device")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = f"cuda:{int(os.environ.get('LOCAL_RANK', 0))}"
    torch.cuda.set_device(device)
    if rank == 0:
        os.makedirs(args.output, exist_ok=True)
        with open(os.path.join(args.output, "args_infer.json"), "w") as f:
            json.dump(vars(args), f, indent=4)
    warn_resolution_mismatch((args.frame_height, args.frame_width))
    hot, _ = evaluate.load_hotpath(args, device)
    model = model_name(args.checkpoint)
    fps = (6 + args.frame_rate) // 2
    results = []
    for i in shard_clips(len(examples), rank, world):
        ex = examples[i]
        g = example_generator(args.seed, i, device)
        input_rgb, batch = prepare_input(args, ex, g, device)
        _, sampled = evaluate.sample_example(hot, batch, args.num_samples, g, args.decoding_t)
        unc, frame_div, mean_div = metrics.sample_diversity(sampled)
        stem = output_stem(args.output, i, ex, model)
        save_results(stem, input_rgb, sampled, unc, (frame_div, mean_div), fps, bool(args.save_images), bool(args.save_mp4),
                     bool(args.save_input), bool(args.save_uncertainty))
        rec = {"example": ex, "index": i, "output": stem, "mean_diversity": float(mean_div)}
        results.append(rec)
        print(json.dumps(rec), flush=True)
    return results


if __name__ == "__main__":
    main()
