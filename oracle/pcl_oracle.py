"""Oracles of the point-cloud conversion (gcd_b200.convert, csrc/unproject.cu) and a seeded writer of synthetic Kubric-4D / ParDom-4D
scene directories.

  unproject_f64   the unprojection in float64 from the same float32 depth and camera rows the kernel reads;
  torch_chain     the reference's float32 torch ops (data-gen/data_utils.py unproject_pixels_to_points + camera_to_world,
                  convert_pcl_kubric.py correct_depth_ball_plane_torch, convert_pcl_pardom.py's clamp), restated op for op on any
                  device, with K and RT built from the camera rows; `.half()` of its result is what the reference stores;
  write_kubric_scene / write_pardom_scene   scene directories as the released datasets lay them out, from a seed.
"""
import json
import os

import numpy as np
import torch

KUBRIC_EDGE = (0.0, -3.0, 40000.0, float("inf"), float("nan"))      # depths the synthetic scenes plant (ParDom adds > 30000 too)


# ---------------------------------------------------------------------------------------------------------------------------
# float64


def unproject_f64(depth, cam, kind, max_depth=30000.0):
    """depth float32 [H, W], cam float32 [16] -> (float64 [H*W, 3] world xyz, float64 [H*W, 3] sum_j |R_ij c_j| + |t_i|, the scale
    of the fp32 rounding error of output i with c the camera-space point). Ball -> plane for kind "kubric", clamp for "pardom"."""
    d = torch.as_tensor(depth).double()
    c = torch.as_tensor(cam).double()
    H, W = d.shape
    fx, fy, cx, cy = c[0], c[1], c[2], c[3]
    R, t = c[4:13].reshape(3, 3), c[13:16]
    u = torch.arange(W, dtype=torch.float64)[None, :].expand(H, W)
    v = torch.arange(H, dtype=torch.float64)[:, None].expand(H, W)
    if kind == "kubric":
        def tans(f, n):
            half = torch.atan(n / (2.0 * f.abs()))
            return torch.tan(-half + 2.0 * half * torch.arange(n, dtype=torch.float64) / max(n - 1, 1))
        mx, my = tans(fx, W), tans(fy, H)
        z = d / torch.sqrt(mx[None, :] ** 2 + my[:, None] ** 2 + 1.0)
    else:
        z = torch.where(torch.isnan(d), d, d.clamp(0.0, max_depth))
    p = torch.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], -1).reshape(-1, 3)
    # the three products summed per row, written out so that 0 * inf gives NaN as in fp32
    ref = torch.stack([p[:, 0] * R[i, 0] + p[:, 1] * R[i, 1] + p[:, 2] * R[i, 2] + t[i] for i in range(3)], -1)
    scale = torch.stack([(p[:, 0] * R[i, 0]).abs() + (p[:, 1] * R[i, 1]).abs() + (p[:, 2] * R[i, 2]).abs() + t[i].abs()
                         for i in range(3)], -1)
    return ref, scale


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's float32 torch chain


def kubric_camera_matrices(row, device):
    c = torch.as_tensor(row, dtype=torch.float32, device=device)
    K = torch.zeros(3, 3, dtype=torch.float32, device=device)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[2, 2] = c[0], c[1], c[2], c[3], 1.0
    RT = torch.eye(4, dtype=torch.float32, device=device)
    RT[0:3, 0:3] = c[4:13].reshape(3, 3)
    RT[0:3, 3] = c[13:16]
    return K, RT


def correct_depth_ball_plane(depth_ball, intrinsics):
    (H, W) = depth_ball.shape[-2:]
    fov_x = 2.0 * torch.atan(W / (2.0 * torch.abs(intrinsics[0, 0])))
    fov_y = 2.0 * torch.atan(H / (2.0 * torch.abs(intrinsics[1, 1])))
    angles_x = torch.linspace(-fov_x / 2.0, fov_x / 2.0, W, dtype=torch.float32, device=depth_ball.device)
    angles_y = torch.linspace(-fov_y / 2.0, fov_y / 2.0, H, dtype=torch.float32, device=depth_ball.device)
    mismatch_x = torch.tan(angles_x)
    mismatch_y = torch.tan(angles_y)
    correction = torch.sqrt(mismatch_x[None, :] ** 2 + mismatch_y[:, None] ** 2 + 1.0)
    return depth_ball / correction


def unproject_points(depth, K, RT):
    (H, W) = depth.shape
    u_coord = torch.arange(W, dtype=torch.float32, device=depth.device)
    v_coord = torch.arange(H, dtype=torch.float32, device=depth.device)
    (u, v) = torch.meshgrid(u_coord, v_coord, indexing="xy")
    z = depth.reshape(-1)
    u = u.reshape(-1)
    v = v.reshape(-1)
    x = (u - K[0, 2]) * z / K[0, 0]
    y = (v - K[1, 2]) * z / K[1, 1]
    xyz_camera = torch.stack((x, y, z), dim=1)
    xyz_world = xyz_camera @ RT[0:3, 0:3].T
    xyz_world += RT[0:3, 3]
    return xyz_world


def torch_chain(depth, cams, kind, device="cpu", max_depth=30000.0):
    """depth float32 [V, H, W], cams float32 [V, 16] -> stored fp16 xyz [V, H*W, 3] (on `device`), view by view as the reference."""
    out = []
    for j in range(depth.shape[0]):
        K, RT = kubric_camera_matrices(cams[j], device)
        d = torch.as_tensor(depth[j], dtype=torch.float32).to(device)
        d = correct_depth_ball_plane(d, K) if kind == "kubric" else torch.clamp(d, 0.0, max_depth)
        out.append(unproject_points(d, K, RT))
    return torch.stack(out).clone().type(torch.float16)


# ---------------------------------------------------------------------------------------------------------------------------
# synthetic scenes


def _look_at_rotation(eye, target=(0.0, 0.0, 0.0)):
    """Camera-to-world rotation (columns: right, down, forward) of a camera at `eye` looking at `target` with z up."""
    f = np.asarray(target, np.float64) - np.asarray(eye, np.float64)
    f /= np.linalg.norm(f)
    r = np.cross(f, [0.0, 0.0, 1.0])
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    return np.stack([r, d, f], 1)


def _quaternion(R):
    """(w, x, y, z) of a rotation matrix (Shepperd's method)."""
    tr = np.trace(R)
    if tr > 0:
        s = 2.0 * np.sqrt(tr + 1.0)
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = 2.0 * np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k])
        q = [0.0] * 4
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    return np.asarray(q)


def _png(path, a, mode):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if mode == "P":
        im = Image.fromarray(a, "P")
        pal = (np.arange(256 * 3, dtype=np.int64) * 37 % 256).astype(np.uint8)
        im.putpalette(pal.tobytes())
    else:
        im = Image.fromarray(a, mode)
    im.save(path)


def _depth_map(rng, H, W, base, edges):
    d = (base * (1.0 + 0.3 * rng.random((H, W)))).astype(np.float32)
    flat = d.reshape(-1)
    idx = rng.choice(H * W, size=len(edges), replace=False)
    flat[idx] = np.asarray(edges, np.float32)
    return d


def _ring(rng, i, V):
    a = 2 * np.pi * (i / V + 0.02 * rng.random())
    rad, hgt = 12.0 + 4.0 * rng.random(), 2.0 + 3.0 * rng.random()
    return np.array([rad * np.cos(a), rad * np.sin(a), hgt])


def write_kubric_scene(root, name, H, W, T, seed):
    """A Kubric-4D scene directory: 16 views of T frames, H x W, cameras on a ring looking at the origin (non-unit quaternions),
    RGBA colour PNGs (RGB on odd views), P-mode segmentation PNGs, float32 depth TIFFs with the KUBRIC_EDGE depths planted; the
    principal point is the image centre, so u == cx on column W / 2. Returns the scene directory."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    scene = os.path.join(root, name)
    os.makedirs(scene, exist_ok=True)
    f = 0.8 + 0.4 * rng.random()
    K = [[f, 0.0, -0.5], [0.0, f * W / H * 1.02, -0.5], [0.0, 0.0, -1.0]]
    for v in range(16):
        eye = _ring(rng, v, 16)
        qs, ps = [], []
        for t in range(T):
            R = _look_at_rotation(eye + 0.05 * t)
            R[:, 1:3] *= -1.0                       # Blender's camera axes: the converter negates columns 1 and 2 back
            qs.append((_quaternion(R) * (0.7 + 0.6 * rng.random())).tolist())
            ps.append((eye + 0.05 * t).tolist())
        meta = {"scene": {"num_frames": T, "resolution": [W, H]}, "camera": {"K": K, "quaternions": qs, "positions": ps}}
        with open(os.path.join(scene, f"{name}_p0_v{v}.json"), "w") as fh:
            json.dump(meta, fh)
        for t in range(T):
            fd = os.path.join(scene, f"frames_p0_v{v}")
            rgba = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            _png(os.path.join(fd, f"rgba_{t:05d}.png"), rgba if v % 2 == 0 else np.ascontiguousarray(rgba[..., :3]),
                 "RGBA" if v % 2 == 0 else "RGB")
            _png(os.path.join(fd, f"segmentation_{t:05d}.png"), rng.integers(0, 12, (H, W), dtype=np.uint8), "P")
            Image.fromarray(_depth_map(rng, H, W, 10.0, KUBRIC_EDGE), "F").save(os.path.join(fd, f"depth_{t:05d}.tiff"))
    return scene


PARDOM_VIEW_NAMES = tuple([f"camera{i}" for i in range(16)] + ["yaw-0", "yaw-60", "yaw-neg-60"])


def write_pardom_scene(root, name, H, W, T, seed, missing=None):
    """A ParDom-4D scene directory: the 19 views (camera0..15, yaw-0, yaw-60, yaw-neg-60) of T frames, H x W, a calibration JSON
    with a lidar entry and non-unit quaternions, RGBA / RGB colour PNGs, P-mode semantic PNGs, npz depth with 0, negative, > 30000,
    +inf and NaN planted. missing = (t, view name): that frame's depth file is not written. Returns the scene directory."""
    rng = np.random.default_rng(seed)
    scene = os.path.join(root, name)
    names, intr, extr = ["velodyne"], [{"fx": 1.0, "fy": 1.0, "cx": 0.0, "cy": 0.0}], \
        [{"rotation": {"qw": 1.0, "qx": 0.0, "qy": 0.0, "qz": 0.0}, "translation": {"x": 0.0, "y": 0.0, "z": 0.0}}]
    for i, vn in enumerate(PARDOM_VIEW_NAMES):
        eye = _ring(rng, i, 19)
        q = _quaternion(_look_at_rotation(eye)) * (0.7 + 0.6 * rng.random())
        f = (0.8 + 0.2 * rng.random()) * W
        names.append(vn)
        intr.append({"fx": f, "fy": f * 1.01, "cx": W / 2.0, "cy": H / 2.0 - 0.25})
        extr.append({"rotation": dict(zip(("qw", "qx", "qy", "qz"), q.tolist())),
                     "translation": dict(zip("xyz", eye.tolist()))})
    os.makedirs(os.path.join(scene, "calibration"), exist_ok=True)
    with open(os.path.join(scene, "calibration", "calib.json"), "w") as fh:
        json.dump({"names": names, "intrinsics": intr, "extrinsics": extr}, fh)
    os.makedirs(os.path.join(scene, "ontology"), exist_ok=True)
    with open(os.path.join(scene, "ontology", "ontology.json"), "w") as fh:
        json.dump({"items": [{"id": i, "name": f"class{i}", "color": dict(zip("rgb", (i * 37 % 256, i * 91 % 256, i * 53 % 256)))}
                             for i in range(256)]}, fh)
    for vn in PARDOM_VIEW_NAMES:
        for t in range(T):
            s = f"{t * 10 + 5:018d}"
            rgba = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            odd = vn.endswith(("1", "3", "5", "7", "9"))
            _png(os.path.join(scene, "rgb", vn, s + ".png"), np.ascontiguousarray(rgba[..., :3]) if odd else rgba,
                 "RGB" if odd else "RGBA")
            _png(os.path.join(scene, "semantic_segmentation_2d", vn, s + ".png"), rng.integers(0, 256, (H, W), dtype=np.uint8),
                 "P")
            if missing is not None and (t, vn) == tuple(missing):
                continue
            os.makedirs(os.path.join(scene, "depth", vn), exist_ok=True)
            np.savez_compressed(os.path.join(scene, "depth", vn, s + ".npz"),
                                data=_depth_map(rng, H, W, 12.0, KUBRIC_EDGE[:2] + (45000.0, 30000.5) + KUBRIC_EDGE[3:]))
    return scene
