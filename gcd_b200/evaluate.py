"""Per-example evaluation of Kubric-4D and ParDom-4D clips on the device: the path of gcd-model/scripts/test.py from the stored
point clouds and a control row to the `*_metrics.json` of one example (SURVEY.md §8(f) rank 3).

    clouds (load_*_clouds) + control row (control_row) -> camera trajectories (kubric_trajectories / pardom_trajectories)
    -> rendered views (gcd_b200.render) -> batch (construct_batch) -> evaluate_example -> save_metrics_json

The host functions reproduce the data modules' deterministic branches (kubric_arbit.py / pardom_arbit.py `sample_trajectories`,
`construct_dict`) operation for operation in numpy / torch float32, so extrinsics, angles, motion buckets and the conditioning noise
equal the reference's bit for bit. The random branches are training-side sampling and raise NotImplementedError.

`evaluate_example` conditions once and samples all S samples of an example as S clips of ONE sampler run, where test.py calls
`sample_video` S times and re-runs the conditioner each time (run_inference, test.py:315-343). The per-step work is the UNet,
sampler and decoder as they are; the once-per-example noise add, last-frame padding and clamps stay torch ops so that the noise
is torch's RNG and reproducible from a `torch.Generator`.

Command line (one `*_metrics.json` per example plus a summary; under torchrun each rank takes `pipeline.shard_clips`):

    python -m gcd_b200.evaluate --kind kubric --checkpoint kubric_gradual_max180.ckpt --examples kubric_test20.txt \\
        --pcl-root /datasets/Kubric-4D/pcl --control-json kubric_valtest_controls_gradual.json --output out/
"""
import argparse
import glob
import json
import math
import os

import numpy as np
import torch

# test.py:474-494: the keys of `calculate_metrics`'s dict in the order it fills them (the last twelve only with a reprojection)
METRIC_KEYS = ("frame_psnr", "frame_ssim", "frame_diversity", "mean_psnr", "mean_ssim", "mean_diversity")
MASKED_METRIC_KEYS = ("frame_psnr_vis", "frame_ssim_vis", "frame_psnr_occ", "frame_ssim_occ", "frame_diversity_vis",
                      "frame_diversity_occ", "mean_psnr_vis", "mean_ssim_vis", "mean_psnr_occ", "mean_ssim_occ",
                      "mean_diversity_vis", "mean_diversity_occ")
LPIPS_KEYS = ("frame_lpips", "mean_lpips")

KUBRIC_FPS, KUBRIC_FRAMES = 24, 60      # kubric_arbit.py:90-92: frames per stored video, and their rate
PARDOM_FPS, PARDOM_FRAMES = 10, 50      # pardom_arbit.py:127-128
PARDOM_WH = (640.0, 480.0)              # ParDom camera resolution: the intrinsics are normalised by it (pardom_arbit.py:555-558)
PARDOM_EGO_POSITION = (1.60, 0.0, 1.55)  # ego_forward camera: position and look-at (pardom_arbit.py:396-400)
PARDOM_EGO_LOOK_AT = (6.60, 0.0, 1.55)
RANDOM = -2222.0                        # test.py:143: control-row angles the data module would sample at random


# ---------------------------------------------------------------------------------------------------------------------------
# readers


def _load_frame_tensors(path, n, what):
    if not os.path.isfile(path):
        raise FileNotFoundError(path)
    obj = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(obj, (list, tuple)) or len(obj) != n or not all(torch.is_tensor(t) for t in obj):
        raise ValueError(f"{path}: expected a list of {n} tensors ({what})")
    return obj


def _stack(frames, path_of, clip_frames):
    try:
        return torch.stack(frames)
    except RuntimeError as e:
        raise ValueError(f"point clouds of frames {list(clip_frames)} under {os.path.dirname(path_of(clip_frames[0]))} differ in "
                         f"shape: {e}") from None


def _check_cloud(path, xyz, rgb, extra=()):
    if xyz.dim() != 3 or xyz.shape[-1] != 3 or rgb.shape != xyz.shape or rgb.dtype != torch.uint8:
        raise ValueError(f"{path}: xyz and rgb must be [V, N, 3] (rgb uint8), got {tuple(xyz.shape)} and {tuple(rgb.shape)} "
                         f"{rgb.dtype}")
    for t in extra:
        if tuple(t.shape) != (*xyz.shape[:2], 1) or t.dtype != torch.uint8:
            raise ValueError(f"{path}: segm / tag must be uint8 [V, N, 1], got {tuple(t.shape)} {t.dtype}")


def kubric_cloud_path(pcl_dir, t):
    return os.path.join(pcl_dir, f"pcl_rgb_segm_{int(t):05d}.pt")


def pardom_cloud_path(pcl_dir, t):
    return os.path.join(pcl_dir, f"pcl_rgb_segm_{int(t) * 10 + 5:06d}.pt")


def load_kubric_clouds(pcl_dir, clip_frames):
    """The stored Kubric-4D clouds of `clip_frames` (kubric_arbit.py:238-260): one file per frame holding [xyz fp16 [V, N, 3],
    rgb uint8 [V, N, 3], segm_rgb uint8 [V, N, 3]]. Returns (xyz fp16 [T, V, N, 3], rgb uint8 [T, V, N, 3]) on the CPU, what
    render.kubric_views takes."""
    xyz, rgb = [], []
    for t in clip_frames:
        p = kubric_cloud_path(pcl_dir, t)
        x, c, s = _load_frame_tensors(p, 3, "xyz, rgb, segm_rgb")
        _check_cloud(p, x, c)
        xyz.append(x.to(torch.float16))
        rgb.append(c)
    path_of = lambda t: kubric_cloud_path(pcl_dir, t)
    return _stack(xyz, path_of, clip_frames), _stack(rgb, path_of, clip_frames)


def load_pardom_clouds(pcl_dir, clip_frames):
    """The stored ParDom-4D clouds of `clip_frames` (pardom_arbit.py:341-368): frame t in `pcl_rgb_segm_{10 t + 5:06d}.pt` holding
    [xyz fp16 [V, N, 3], rgb uint8 [V, N, 3], segm uint8 [V, N, 1], tag uint8 [V, N, 1]]. Returns (xyz [T, V, N, 3], rgb
    [T, V, N, 3], segm [T, V, N, 1]) on the CPU, what render.pardom_views takes (the view tags are not used by the renderer)."""
    xyz, rgb, segm = [], [], []
    for t in clip_frames:
        p = pardom_cloud_path(pcl_dir, t)
        x, c, s, tag = _load_frame_tensors(p, 4, "xyz, rgb, segm, tag")
        _check_cloud(p, x, c, (s, tag))
        xyz.append(x.to(torch.float16))
        rgb.append(c)
        segm.append(s)
    path_of = lambda t: pardom_cloud_path(pcl_dir, t)
    return _stack(xyz, path_of, clip_frames), _stack(rgb, path_of, clip_frames), _stack(segm, path_of, clip_frames)


def read_kubric_intrinsics(scene_dir):
    """Normalised intrinsics [3, 3] float32 of the scene's stored view 4 (`<scene>_p0_v4.json`, the view the control rows'
    source trajectory starts at; kubric_arbit.py:171-174, geometry.py:56-57: |K|)."""
    name = os.path.basename(os.path.normpath(scene_dir))
    with open(os.path.join(scene_dir, f"{name}_p0_v4.json")) as f:
        K = json.load(f)["camera"]["K"]
    K = torch.tensor(np.abs(np.asarray(K, dtype=np.float64)), dtype=torch.float32)
    if K.shape != (3, 3):
        raise ValueError(f"{scene_dir}: camera K must be 3 x 3, got {tuple(K.shape)}")
    return K


def read_pardom_intrinsics(scene_dir):
    """Pixel intrinsics [V, 3, 3] float32 of the scene's cameras, sorted by name without the lidar (calibration/*.json;
    geometry.py:95-131)."""
    paths = sorted(glob.glob(os.path.join(scene_dir, "calibration", "*.json")))
    if not paths:
        raise FileNotFoundError(os.path.join(scene_dir, "calibration", "*.json"))
    with open(paths[0]) as f:
        cal = json.load(f)
    K = {n: torch.tensor([[i["fx"], 0.0, i["cx"]], [0.0, i["fy"], i["cy"]], [0.0, 0.0, 1.0]], dtype=torch.float32)
         for n, i in zip(cal["names"], cal["intrinsics"]) if "velodyne" not in n.lower()}
    return torch.stack([K[n] for n in sorted(K)])


def read_pardom_palette(ontology_path):
    """The semantic-id colours [256, 3] float32 in [0, 1] of a ParDom ontology file (pardom_arbit.py:136-144)."""
    with open(ontology_path) as f:
        items = json.load(f)["items"]
    pal = torch.zeros(256, 3, dtype=torch.float64)
    for x in items:
        pal[int(x["id"])] = torch.tensor([x["color"]["r"], x["color"]["g"], x["color"]["b"]], dtype=torch.float64) / 255.0
    return pal.to(torch.float32)


def load_pardom_ego_frames(scene_dir, clip_frames, frame_hw=(256, 384), modality="rgb"):
    """The forward ego camera's stored frames (`<scene>/rgb/yaw-0/{10 t + 5:018d}.png`, the `ego_forward` input of
    pardom_arbit.py:314-327): centre crop to the frame aspect, bilinear resize, `* 2 - 1`. Returns float32 [T, 3, H, W]. The
    reference resizes with cv2 INTER_LINEAR; torch's bilinear resize without antialiasing uses the same weights, the sums may
    round differently in the last bit."""
    if modality != "rgb":
        raise NotImplementedError(f"ego input modality {modality!r}: only rgb is read")
    from torchvision.io import decode_png, read_file
    H, W = frame_hw
    out = []
    for t in clip_frames:
        img = decode_png(read_file(os.path.join(scene_dir, "rgb", "yaw-0", f"{int(t) * 10 + 5:018d}.png")))[:3]
        x = img.to(torch.float32) / 255.0
        h, w = x.shape[-2:]
        ar = W / H
        if w / h > ar + 2e-3:
            cw = int(h * ar)
            x = x[:, :, (w - cw) // 2:(w - cw) // 2 + cw]
        elif w / h < ar - 2e-3:
            ch = int(w / ar)
            x = x[:, (h - ch) // 2:(h - ch) // 2 + ch, :]
        if tuple(x.shape[-2:]) != (H, W):
            x = torch.nn.functional.interpolate(x[None], (H, W), mode="bilinear", align_corners=False)[0]
        out.append(x * 2.0 - 1.0)
    return torch.stack(out)


# ---------------------------------------------------------------------------------------------------------------------------
# control rows and clip frames


def control_row(kind, entry=None, frame_start=-1, frame_stride=-1, frame_rate=-1, angles=None):
    """A row [frame_start, frame_stride, frame_rate, az0, az1, el0, el1, r0, r1] (float32, degrees) as load_input_gt builds it
    (test.py:135-191, 242-261). `entry`: one `sample_XX` dict of a controls JSON (eval/list/*_valtest_controls*.json): its frame
    bounds fill the negative arguments and, for Kubric, its spherical_start / spherical_end set the angles. Without an entry the
    frame arguments are required; `angles` = (azimuth_start, delta_azimuth, elevation_start, delta_elevation, radius_start,
    delta_radius) gives the Kubric trajectory explicitly (test.py's --azimuth_start ... options), None leaves it to random
    sampling. ParDom rows carry no angles."""
    if kind not in ("kubric", "pardom"):
        raise ValueError(f"unknown dataset kind {kind!r}")
    if angles is not None:
        if len(angles) != 6:
            raise ValueError("angles: (azimuth_start, delta_azimuth, elevation_start, delta_elevation, radius_start, delta_radius)")
        a0, da, e0, de, r0, dr = (float(a) for a in angles)
        row = np.array([frame_start, frame_stride, frame_rate, a0, a0 + da, e0, e0 + de, r0, r0 + dr], dtype=np.float32)
    else:
        row = np.array([frame_start, frame_stride, frame_rate] + [RANDOM] * 6, dtype=np.float32)
    if kind == "pardom":
        row[3:9] = 0.0
    if entry is None:
        if frame_start < 0 or frame_stride < 0 or frame_rate < 0:
            raise ValueError("without a controls entry, frame_start, frame_stride and frame_rate must all be given")
        return row
    try:
        if kind == "kubric":
            s0, s1 = entry["spherical_start"], entry["spherical_end"]
            row[3:9] = [s0[0], s1[0], s0[1], s1[1], s0[2], s1[2]]
        if frame_start < 0:
            row[0] = entry["frame_start"]
        if frame_stride < 0:
            row[1] = entry["frame_skip"]
    except (KeyError, IndexError, TypeError) as e:
        raise ValueError(f"malformed controls entry: {e!r}") from None
    if frame_rate < 0:
        row[2] = int(round((KUBRIC_FPS if kind == "kubric" else PARDOM_FPS) / row[1]))
    return row


def control_entry(control_info, example, control_idx=0):
    """`control_info[<scene>]["sample_XX"]` of a loaded controls JSON for an example path (test.py:177-178, 253-254)."""
    name = os.path.basename(os.path.normpath(example))
    try:
        return control_info[name][f"sample_{control_idx:02d}"]
    except KeyError:
        raise KeyError(f"controls JSON has no entry {name}/sample_{control_idx:02d}") from None


def clip_frames(kind, row, num_frames=14):
    """(frame indices [T] int64, fps) of a control row: stride apart from frame_start, within the stored video
    (kubric_arbit.py:159-162, pardom_arbit.py:215-218); fps = round(stored rate / stride)."""
    rate, avail = (KUBRIC_FPS, KUBRIC_FRAMES) if kind == "kubric" else (PARDOM_FPS, PARDOM_FRAMES)
    start, stride = int(row[0]), int(row[1])
    if stride < 1 or start < 0:
        raise ValueError(f"frame_start {start} and frame_stride {stride}: need start >= 0 and stride >= 1")
    frames = np.arange(num_frames) * stride + start
    if frames[-1] > avail - 1:
        raise ValueError(f"clip frames {frames[0]}..{frames[-1]} run past the {avail} stored frames")
    return frames, int(round(rate / stride))


# ---------------------------------------------------------------------------------------------------------------------------
# camera trajectories


def _alpha(trajectory, t, move_time):
    if trajectory == "interpol_linear":
        return t / move_time
    if trajectory == "interpol_sine":
        return (1.0 - np.cos(t / move_time * np.pi)) / 2.0
    raise ValueError(f"Unknown trajectory: {trajectory}")


def _look_at(position, target):
    """Camera pose [4, 4] (columns right, down, forward; translation = position) looking from `position` at `target`, world up +z
    (geometry.py:192-217)."""
    fwd = target - position
    fwd /= np.linalg.norm(fwd)
    right = np.cross(np.array([0, 0, -1]), fwd)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    RT = np.eye(4)
    RT[0:3, 0:3] = np.stack([right, down, fwd], axis=1)
    RT[0:3, 3] = position
    return RT


def _poses(positions, targets):
    out = np.zeros((len(positions), 4, 4), dtype=np.float32)
    for t in range(len(positions)):
        out[t] = _look_at(positions[t], targets[t])
    return torch.tensor(out, dtype=torch.float32)


def _cartesian_deg(sph):
    az, el, r = np.deg2rad(sph[..., 0]), np.deg2rad(sph[..., 1]), sph[..., 2]
    return np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], axis=-1)


def _check_move_time(move_time, num_frames):
    if not 0 <= move_time <= num_frames:
        raise ValueError(f"move_time {move_time} must lie in [0, {num_frames}]")


def kubric_trajectories(row, num_frames=14, trajectory="interpol_linear", move_time=13, delta_azimuth_range=(-180.0, 180.0),
                        delta_elevation_range=(-60.0, 60.0)):
    """Source and target cameras of a Kubric-4D control row (the deterministic branch of kubric_arbit.py:262-409): the source
    camera stays at the start angles, the target moves to the end angles over the first `move_time` frames (`trajectory`
    interpolation), both on the sphere around (0, 0, 1) looking at it. Defaults: the gradual max-180 configs; the max-90 ones
    use delta ranges (-90, 90) / (-30, 30), the direct ones move_time 0.

    Returns dict: spherical_src / spherical_dst float32 [T, 3] (degrees, degrees, radius), extrinsics_src / extrinsics_dst
    float32 [T, 4, 4], motion_amount (float, the angular distance over the configured maximum; sets the motion bucket)."""
    row = np.asarray(row, dtype=np.float32)
    if row.shape != (9,):
        raise ValueError(f"a control row has 9 values, got shape {row.shape}")
    if not row[3] > -1000:
        raise NotImplementedError("random Kubric trajectory sampling (range sampling of kubric_arbit.py:285-357) is training-side; "
                                  "give the angles in the control row")
    _check_move_time(move_time, num_frames)
    start = np.array([float(row[3]), float(row[5]), float(row[7])], dtype=np.float32)
    end = np.array([float(row[4]), float(row[6]), float(row[8])], dtype=np.float32)
    motion = np.linalg.norm(end[0:2] - start[0:2], ord=2)
    motion_max = np.linalg.norm([max(*delta_azimuth_range), max(*delta_elevation_range)], ord=2)
    src = np.tile(start[None], (num_frames, 1))
    dst = np.tile(end[None], (num_frames, 1))
    for t in range(move_time):
        a = _alpha(trajectory, t, move_time)
        dst[t] = start * (1.0 - a) + end * a
    pos_src, pos_dst = _cartesian_deg(src), _cartesian_deg(dst)
    pos_src[..., 2] += 1.0
    pos_dst[..., 2] += 1.0
    centre = np.tile(np.array([0.0, 0.0, 1.0], dtype=np.float32)[None], (num_frames, 1))
    return dict(spherical_src=torch.tensor(src, dtype=torch.float32), spherical_dst=torch.tensor(dst, dtype=torch.float32),
                extrinsics_src=_poses(pos_src, centre), extrinsics_dst=_poses(pos_dst, centre), motion_amount=motion / motion_max)


def pardom_trajectories(intrinsics, num_frames=14, input_mode="ego_forward", output_mode="topdown1",
                        dst_cam_position=(-8.0, 0.0, 8.0), dst_cam_look_at=(5.6, 0.0, 1.55), dst_azimuth_range=(0.0, 0.0),
                        trajectory="interpol_sine", move_time=13):
    """Source and target cameras of a ParDom-4D clip (pardom_arbit.py:369-562) in the modes every shipped config uses:
    `ego_forward` input (the forward ego camera) and `topdown1` output (a fixed camera behind and above the car at
    `dst_cam_position` looking at `dst_cam_look_at`), reached from the ego camera over the first `move_time` frames. No random
    numbers are drawn. Defaults: the gradual configs; the direct ones use move_time 0.

    intrinsics: float32 [V, 3, 3] pixel intrinsics of the scene's cameras in name order (read_pardom_intrinsics); the
    second-to-last camera's are used for both trajectories, as the reference does.
    Returns dict: extrinsics_src / extrinsics_dst float32 [T, 4, 4], intrinsics_src / intrinsics_dst float32 [T, 3, 3]
    normalised to [0, 1]^2, readable_angles float32 [T, 3] (zeros), motion_amount 0.5."""
    if input_mode != "ego_forward" or output_mode != "topdown1":
        raise NotImplementedError(f"ParDom input_mode {input_mode!r} / output_mode {output_mode!r}: only ego_forward -> topdown1 is "
                                  "built (magic_random, topdown2 and traffic1 sample at random; magic_opposite reads stored frames)")
    if list(dst_azimuth_range) != [0.0, 0.0]:
        raise ValueError(f"topdown1 takes no azimuth range, got {list(dst_azimuth_range)}")
    intrinsics = torch.as_tensor(intrinsics)
    if intrinsics.dim() != 3 or intrinsics.shape[0] < 2 or tuple(intrinsics.shape[1:]) != (3, 3):
        raise ValueError(f"intrinsics must be [V >= 2, 3, 3], got {tuple(intrinsics.shape)}")
    _check_move_time(move_time, num_frames)
    T = num_frames
    tile = lambda v: np.tile(np.array(v, dtype=np.float32)[None], (T, 1))
    pos_src, look_src = tile(PARDOM_EGO_POSITION), tile(PARDOM_EGO_LOOK_AT)
    pos_dst, look_dst = tile(dst_cam_position), tile(dst_cam_look_at)
    K_src = intrinsics.to(torch.float32)[-2:-1].tile((T, 1, 1))
    K_dst = intrinsics.to(torch.float32)[-2:-1].tile((T, 1, 1))
    for t in range(move_time):
        p0, p1, l0, l1 = pos_src[t].copy(), pos_dst[t].copy(), look_src[t].copy(), look_dst[t].copy()
        k0, k1 = K_src[t].clone(), K_dst[t].clone()
        a = _alpha(trajectory, t, move_time)
        pos_dst[t] = p0 * (1.0 - a) + p1 * a
        look_dst[t] = l0 * (1.0 - a) + l1 * a
        K_dst[t] = k0 * (1.0 - a) + k1 * a
    out = dict(extrinsics_src=_poses(pos_src, look_src), extrinsics_dst=_poses(pos_dst, look_dst),
               readable_angles=torch.zeros(T, 3, dtype=torch.float32), motion_amount=0.5)
    for K in (K_src, K_dst):
        K[:, 0, :] /= PARDOM_WH[0]
        K[:, 1, :] /= PARDOM_WH[1]
    out.update(intrinsics_src=K_src, intrinsics_dst=K_dst)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# batch


def _pad_last(frames, keep, T):
    if keep < T:
        frames = torch.cat([frames[0:keep]] + [frames[keep - 1:keep]] * (T - keep), dim=0)
    return frames


def construct_batch(kind, traj, rgb_src, rgb_dst, reproject, fps, generator, cond_aug=0.02, motion_bucket_range=None,
                    input_frames=None, output_frames=None):
    """The model batch of one example (construct_dict, kubric_arbit.py:565-647 / pardom_arbit.py:740-826).

    traj: the dict of kubric_trajectories / pardom_trajectories; rgb_src / rgb_dst / reproject: [T, 3, H, W] in [-1, 1] on any
    device (reproject may be None); fps: the clip's frame rate (clip_frames); generator: the torch.Generator the conditioning
    noise is drawn from, on its own device (a CPU generator draws what the reference's `torch.randn` draws on the CPU);
    motion_bucket_range: (lo, hi), default (0, 255) for Kubric and (127, 127) for ParDom as the shipped configs set it;
    input_frames / output_frames: frames kept before the last one is repeated (default T: none).

    Returns dict: cond_aug float32 [T], motion_bucket_id / fps_id int32 [T], image_only_indicator float32 [1, T],
    scaled_relative_pose float32 [T, 3, 4] (inv(RT_src) @ RT_dst), scaled_relative_angles float32 [T, 3] (Kubric: target minus
    source spherical angles with azimuth / elevation in radians; ParDom: the readable angles), and on rgb_src's device jpg,
    cond_frames_without_noise, cond_frames = cond_frames_without_noise + cond_aug * randn (+ reproject), float32 [T, 3, H, W]."""
    if kind not in ("kubric", "pardom"):
        raise ValueError(f"unknown dataset kind {kind!r}")
    ext_src, ext_dst = traj["extrinsics_src"], traj["extrinsics_dst"]
    T = ext_src.shape[0]
    if motion_bucket_range is None:
        motion_bucket_range = (0, 255) if kind == "kubric" else (127, 127)
    lo, hi = motion_bucket_range
    if hi - lo <= 0:
        motion_value = int(lo)
    else:
        motion_value = int(round(lo + (hi - lo) * traj["motion_amount"]))
    rel_pose = torch.zeros((T, 3, 4), dtype=torch.float32)
    for t in range(T):
        rel_pose[t] = (torch.linalg.inv(ext_src[t]) @ ext_dst[t])[0:3, 0:4]
    if kind == "kubric":
        angles = traj["spherical_dst"] - traj["spherical_src"]
        angles[:, 0] *= torch.pi / 180.0
        angles[:, 1] *= torch.pi / 180.0
    else:
        angles = traj["readable_angles"].clone()
    batch = dict(cond_aug=torch.ones((T,), dtype=torch.float32) * cond_aug,
                 motion_bucket_id=torch.ones((T,), dtype=torch.int32) * motion_value,
                 fps_id=torch.ones((T,), dtype=torch.int32) * int(fps),
                 image_only_indicator=torch.zeros((1, T), dtype=torch.float32),
                 scaled_relative_pose=rel_pose, scaled_relative_angles=angles.to(torch.float32))
    target = _pad_last(rgb_dst, T if output_frames is None else output_frames, T)
    cond = _pad_last(rgb_src, T if input_frames is None else input_frames, T)
    if target.shape != cond.shape or target.shape[0] != T:
        raise ValueError(f"target {tuple(target.shape)} and conditioning {tuple(cond.shape)} frames must both be [{T}, 3, H, W]")
    noise = torch.randn(*cond.shape, generator=generator, device=generator.device)
    batch.update(jpg=target.to(torch.float32), cond_frames=(cond + cond_aug * noise.to(cond.device)).to(torch.float32),
                 cond_frames_without_noise=cond.to(torch.float32))
    if reproject is not None:
        batch["reproject"] = reproject.to(torch.float32)
    return batch


# ---------------------------------------------------------------------------------------------------------------------------
# sampling and metrics


@torch.no_grad()
def sample_example(hotpath, batch, num_samples, generator, decoding_t=14, num_steps=None):
    """Conditions once and samples all S samples of one example as S clips of one sampler run, then decodes each clip.

    hotpath: a gcd_b200.pipeline.GCDHotPath with its conditioner loaded (load_clip, load_cond_encoder, and load_spherical for a
    Kubric UNet); batch: a construct_batch dict; generator: the latent noise of sample s is the s-th `randn([T, 4, H/8, W/8])`
    drawn from it, on its device (what the s-th sequential sample_video call draws from the device RNG); decoding_t: frames per
    decoder chunk. (c, uc) are repeated S times and the S samples are S clips of one sample_latents call (test.py / infer.py call
    sample_video S times and re-run the conditioner each time).

    Returns (samples, sampled): samples a list of S dicts {cond_rgb, sampled_rgb [T, 3, H, W] in [0, 1], sampled_latent
    [T, 4, H/8, W/8]}, sampled the stacked sampled_rgb [S, T, 3, H, W], all on the device."""
    if num_samples < 1:
        raise ValueError(f"num_samples must be >= 1, got {num_samples}")
    dev = hotpath.device
    T = hotpath.T
    cond_frames = batch["cond_frames"].to(dev)
    if cond_frames.shape[0] != T:
        raise ValueError(f"the batch holds {cond_frames.shape[0]} frames; the pipeline samples clips of {T}")
    _, _, H, W = cond_frames.shape
    c, uc = hotpath.condition(batch)
    rep = lambda d: {k: v.repeat(num_samples, *([1] * (v.dim() - 1))) for k, v in d.items()}
    noise = torch.cat([torch.randn((T, 4, H // 8, W // 8), generator=generator, device=generator.device)
                       for _ in range(num_samples)]).to(dev, torch.float32)
    z = hotpath.sample_latents(noise, rep(c), rep(uc), num_steps)
    x = torch.cat([hotpath.decode_first_stage(z[s * T:(s + 1) * T], decoding_t) for s in range(num_samples)])
    sampled = torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0).view(num_samples, T, 3, H, W)
    cond_rgb = torch.clamp((cond_frames + 1.0) / 2.0, min=0.0, max=1.0)
    samples = [dict(cond_rgb=cond_rgb, sampled_rgb=sampled[s], sampled_latent=z[s * T:(s + 1) * T]) for s in range(num_samples)]
    return samples, sampled


@torch.no_grad()
def evaluate_example(hotpath, views, batch, num_samples, generator, lpips=None, decoding_t=14, num_steps=None):
    """test.py's run_inference + calculate_metrics for one example, with all samples in one sampler run (sample_example).

    views: (gt, reproject), the target video and the reprojection baseline [T, 3, H, W] in [-1, 1] (batch["jpg"],
    batch.get("reproject")); lpips: optional gcd_b200.lpips.LPIPS (adds frame_lpips / mean_lpips to the metrics); the other
    arguments as sample_example's.

    Returns (samples, metrics, uncertainty): samples as sample_example's, metrics calculate_metrics's dict (CPU tensors),
    uncertainty [T, H, W] on the device."""
    from . import metrics
    samples, sampled = sample_example(hotpath, batch, num_samples, generator, decoding_t, num_steps)
    gt, reproject = views
    dev = hotpath.device
    gt01 = (gt.to(dev, torch.float32) + 1.0) / 2.0
    rep01 = None if reproject is None else (reproject.to(dev, torch.float32) + 1.0) / 2.0
    m, unc = metrics.calculate_metrics(gt01, rep01, sampled, lpips=lpips)
    return samples, m, unc


def save_metrics_json(path, metrics):
    """Writes a metrics dict as test.py does (test.py:876, eval_utils.save_json): keys in the reference's order, arrays as nested
    lists, scalars as numbers, NaN as NaN, indent 4."""
    order = METRIC_KEYS + MASKED_METRIC_KEYS + LPIPS_KEYS
    keys = [k for k in order if k in metrics] + [k for k in metrics if k not in order]
    out = {}
    for k in keys:
        v = metrics[k]
        if torch.is_tensor(v):
            v = v.detach().cpu().tolist()
        elif isinstance(v, np.ndarray):
            v = v.tolist()
        elif isinstance(v, (np.floating, np.integer)):
            v = v.item()
        out[k] = v
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=4)


# ---------------------------------------------------------------------------------------------------------------------------
# command line


def _model_config(path, kind):
    from . import spec
    cfg = {}
    if path:
        with open(path) as f:
            cfg = json.load(f)
        unknown = set(cfg) - {"unet", "vae", "encoder", "vit"}
        if unknown:
            raise ValueError(f"{path}: unknown sections {sorted(unknown)} (unet, vae, encoder, vit)")
    unet = dict(spec.UNET_KUBRIC if kind == "kubric" else spec.UNET_PARDOM, **cfg.get("unet", {}))
    return unet, dict(spec.VAE_DECODER, **cfg.get("vae", {})), dict(spec.VAE_ENCODER, **cfg.get("encoder", {})), cfg.get("vit")


def load_hotpath(args, device):
    """A GCDHotPath with UNet, decoder and conditioner, and an LPIPS model when the checkpoint holds its weights, all loaded from
    one checkpoint through checkpoint.HotPathRoot."""
    from . import checkpoint, embedders, spec
    from .lpips import LPIPS
    from .pipeline import GCDHotPath
    from .unet import VideoUNet
    from .vae import VideoDecoder
    ucfg, vcfg, ecfg, vit = _model_config(args.model_config, args.kind)
    spherical = bool(ucfg.get("aux_emb_dim", 0))
    unet = VideoUNet(**spec.unet_ctor_kwargs(ucfg))
    dec = VideoDecoder(**spec.decoder_ctor_kwargs(vcfg))
    embs = embedders.build_embedders(embedders.gcd_conditioner_config(spherical=spherical, vit_cfg=vit, enc_cfg=ecfg))
    lp = LPIPS()
    root = checkpoint.HotPathRoot(unet, dec, conditioner=embs, lpips=lp)
    missing, _ = root.init_from_ckpt(args.checkpoint, use_ema=bool(args.use_ema))
    lp_missing = [k for k in missing if k.startswith("lpips.")]
    missing = [k for k in missing if not k.startswith("lpips.")]
    if missing:
        raise KeyError(f"{args.checkpoint} lacks {len(missing)} tensors of the evaluated model, e.g. {missing[:5]}")
    if lp_missing and len(lp_missing) != len(list(lp.state_dict())):
        raise KeyError(f"{args.checkpoint} holds some but not all LPIPS tensors, e.g. missing {lp_missing[:5]}")
    hot = GCDHotPath(ucfg, vcfg, num_steps=args.num_steps, num_frames=args.num_frames, max_scale=args.guider_max_scale,
                     min_scale=args.guider_min_scale, device=device, unet=unet.to(device), decoder=dec.to(device))
    hot.load_clip(embs[0].open_clip.state_dict(), vit_cfg=vit)
    ae = embs[3].encoder
    hot.load_cond_encoder(ae.encoder.state_dict(), ae.quant_conv.weight.detach(), ae.quant_conv.bias.detach(), enc_cfg=ecfg)
    if spherical:
        hot.load_spherical(embs[5].proj.weight.detach(), embs[5].proj.bias.detach())
    return hot, (None if lp_missing else lp.to(device))


def prepare_example(args, example, control_info, generator, device):
    """Clouds, trajectories, rendered views and batch of one example. Returns (views, batch)."""
    from . import render
    entry = control_entry(control_info, example, args.control_idx) if control_info is not None else None
    angles = None
    if args.azimuth_start is not None:
        angles = (args.azimuth_start, args.delta_azimuth, args.elevation_start, args.delta_elevation, args.radius_start,
                  args.delta_radius)
    row = control_row(args.kind, entry, args.frame_start, args.frame_stride, args.frame_rate, angles)
    frames, fps = clip_frames(args.kind, row, args.num_frames)
    name = os.path.basename(os.path.normpath(example))
    pcl_dir = os.path.join(args.pcl_root, name)
    hw = dict(render_hw=(args.render_height, args.render_width), frame_hw=(args.frame_height, args.frame_width))
    move_time = args.move_time
    if args.kind == "kubric":
        traj = kubric_trajectories(row, args.num_frames, args.trajectory or "interpol_linear", 13 if move_time is None else move_time,
                                   (-args.max_delta_azimuth, args.max_delta_azimuth),
                                   (-args.max_delta_elevation, args.max_delta_elevation))
        xyz, rgb = load_kubric_clouds(pcl_dir, frames)
        src, dst, rep = render.kubric_views(xyz.to(device), rgb.to(device), read_kubric_intrinsics(example),
                                            traj["extrinsics_src"], traj["extrinsics_dst"], reproject=True, **hw)
    else:
        traj = pardom_trajectories(read_pardom_intrinsics(example), args.num_frames,
                                   trajectory=args.trajectory or "interpol_sine", move_time=13 if move_time is None else move_time)
        xyz, rgb, segm = load_pardom_clouds(pcl_dir, frames)
        palette = None
        if args.modality == "segm":
            palette = read_pardom_palette(args.ontology).to(device)
        dst, rep = render.pardom_views(xyz.to(device), rgb.to(device), traj["intrinsics_dst"], traj["extrinsics_dst"],
                                       args.modality, segm.to(device), palette, 0, True, **hw)
        src = load_pardom_ego_frames(example, frames, hw["frame_hw"]).to(device)
    batch = construct_batch(args.kind, traj, src, dst, rep, fps, generator, cond_aug=args.cond_aug,
                            motion_bucket_range=args.motion_bucket_range)
    return (batch["jpg"], batch.get("reproject")), batch


def read_examples(path):
    with open(path) as f:
        return [ln.strip() for ln in f if ln.strip() and not ln.strip().startswith("#")]


def summarize(results):
    """Mean over examples of each per-example mean (NaN-aware, as np.nanmean): mean_* metrics averaged over samples first."""
    out = {"examples": len(results)}
    keys = [k for k in results[0] if k.startswith("mean_")] if results else []
    for k in keys:
        vals = [float(np.nanmean(np.asarray(r[k], dtype=np.float64))) for r in results if k in r]
        vals = [v for v in vals if not math.isnan(v)]
        out[k] = sum(vals) / len(vals) if vals else float("nan")
    return out


def parser():
    p = argparse.ArgumentParser(prog="python -m gcd_b200.evaluate",
                                description="Evaluate a GCD checkpoint on Kubric-4D / ParDom-4D examples (test.py's metrics, no videos).")
    p.add_argument("--kind", choices=["kubric", "pardom"], required=True)
    p.add_argument("--checkpoint", required=True, help=".ckpt or .safetensors with the DiffusionEngine's keys")
    p.add_argument("--use-ema", type=int, default=0)
    p.add_argument("--model-config", default="", help="JSON with unet / vae / encoder / vit overrides of the GCD shapes")
    p.add_argument("--examples", required=True, help="text file with one scene directory per line (eval/list/*_test*.txt)")
    p.add_argument("--pcl-root", required=True, help="directory holding <scene>/pcl_rgb_segm_*.pt")
    p.add_argument("--control-json", default="")
    p.add_argument("--control-idx", type=int, default=0)
    p.add_argument("--output", required=True)
    p.add_argument("--num-samples", type=int, default=2)
    p.add_argument("--num-frames", type=int, default=14)
    p.add_argument("--num-steps", type=int, default=25)
    p.add_argument("--guider-max-scale", type=float, default=1.5)
    p.add_argument("--guider-min-scale", type=float, default=1.0)
    p.add_argument("--cond-aug", type=float, default=0.02)
    p.add_argument("--decoding-t", type=int, default=14)
    p.add_argument("--seed", type=int, default=0, help="seeds the device generator of the conditioning and latent noise")
    p.add_argument("--frame-start", type=int, default=-1)
    p.add_argument("--frame-stride", type=int, default=-1)
    p.add_argument("--frame-rate", type=int, default=-1)
    p.add_argument("--azimuth-start", type=float, default=None, help="Kubric angles without a control JSON")
    p.add_argument("--delta-azimuth", type=float, default=30.0)
    p.add_argument("--elevation-start", type=float, default=10.0)
    p.add_argument("--delta-elevation", type=float, default=15.0)
    p.add_argument("--radius-start", type=float, default=15.0)
    p.add_argument("--delta-radius", type=float, default=0.0)
    p.add_argument("--trajectory", choices=["interpol_linear", "interpol_sine"], default=None,
                   help="default: interpol_linear for Kubric, interpol_sine for ParDom")
    p.add_argument("--move-time", type=int, default=None, help="frames the target camera moves over (gradual 13, direct 0)")
    p.add_argument("--max-delta-azimuth", type=float, default=180.0, help="Kubric motion normalisation (max-90 configs: 90)")
    p.add_argument("--max-delta-elevation", type=float, default=60.0, help="Kubric motion normalisation (max-90 configs: 30)")
    p.add_argument("--motion-bucket-range", type=int, nargs=2, default=None)
    p.add_argument("--modality", choices=["rgb", "segm"], default="rgb", help="ParDom output modality")
    p.add_argument("--ontology", default="", help="ParDom ontology JSON (segm modality)")
    p.add_argument("--frame-height", type=int, default=256)
    p.add_argument("--frame-width", type=int, default=384)
    p.add_argument("--render-height", type=int, default=280)
    p.add_argument("--render-width", type=int, default=420)
    return p


def main(argv=None):
    from .pipeline import shard_clips
    args = parser().parse_args(argv)
    if args.modality == "segm" and not args.ontology:
        raise SystemExit("--modality segm needs --ontology")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if not torch.cuda.is_available():
        raise SystemExit("gcd_b200.evaluate runs on a CUDA device")
    device = f"cuda:{local}"
    torch.cuda.set_device(device)
    examples = read_examples(args.examples)
    control_info = None
    if args.control_json:
        with open(args.control_json) as f:
            control_info = json.load(f)
    hot, lp = load_hotpath(args, device)
    mine = shard_clips(len(examples), rank, world)
    results = []
    for i in mine:
        ex = examples[i]
        g = torch.Generator(device=device).manual_seed(args.seed * 1000003 + i)
        views, batch = prepare_example(args, ex, control_info, g, device)
        _, m, _ = evaluate_example(hot, views, batch, args.num_samples, g, lpips=lp, decoding_t=args.decoding_t)
        name = os.path.basename(os.path.normpath(ex))
        path = os.path.join(args.output, f"{i:03d}_{name}_c{args.control_idx:02d}_metrics.json")
        save_metrics_json(path, m)
        results.append({k: v for k, v in m.items() if k.startswith("mean_")})
        print(json.dumps({"example": name, "index": i, "metrics": path,
                          "mean_psnr": float(np.nanmean(m["mean_psnr"].numpy())),
                          "mean_ssim": float(np.nanmean(m["mean_ssim"].numpy()))}), flush=True)
    summary = summarize(results)
    summary.update(rank=rank, world=world, num_samples=args.num_samples, checkpoint=os.path.basename(args.checkpoint))
    save_metrics_json(os.path.join(args.output, f"summary_rank{rank}.json"), summary)
    print(json.dumps(summary), flush=True)
    return summary


if __name__ == "__main__":
    main()
