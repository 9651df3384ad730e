"""Writes tests/golden/pcl_kubric.pt and tests/golden/pcl_pardom.pt from the reference's own conversion code (needs a reference
checkout: GCD_REFERENCE, see oracle/ref_shim.py; the scripts are in its data-gen directory) and asserts oracle/pcl_oracle.py's torch
chain against it bit for bit.

    python -m oracle.pin_convert

Cut out of the reference sources with `ast` (oracle/pin_evaluate.py's `_cut`) and run on CPU over seeded synthetic scenes
(oracle/pcl_oracle.write_*_scene, written to a temporary directory):
  data-gen/convert_pcl_kubric.py   is_finished, get_kubric_camera_matrices_torch, correct_depth_ball_plane_torch, process_example;
  data-gen/convert_pcl_pardom.py   is_finished, get_intrinsics_matrix, get_extrinsics_matrix, process_example;
  data-gen/data_utils.py           load_json, camera_to_world, unproject_pixels_to_points.
Two names are replaced because their libraries are not installed: `Quaternion(...).rotation_matrix` by
gcd_b200.convert.quaternion_rotation_matrix (pyquaternion's formula restated in float64) and `plt.imread` by `_mpl_imread` below
(matplotlib's PNG rule for 8-bit RGB / RGBA / P / LA: np.divide(bytes, 255, dtype=float32), P and LA through RGBA). The one source
edit is `device = torch.device(f'cuda:{gpu_idx}')` -> `device = 'cpu'`. All three are recorded in the goldens' metadata.
Scenes are regenerated from their seeds; only the reference's stored lists are kept.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import convert as C  # noqa: E402
from oracle import pcl_oracle as P  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.pin_evaluate import _cut  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
DEVICE_EDIT = ("device = torch.device(f'cuda:{gpu_idx}')", "device = 'cpu'")
T = 3
KUBRIC = dict(kind="kubric", name="scn00007", H=12, W=16, T=T, seed=31)
PARDOM = dict(kind="pardom", name="scene_000007", H=12, W=16, T=T, seed=32, missing=(1, "camera3"))


def write_case(root, c):
    if c["kind"] == "kubric":
        return P.write_kubric_scene(root, c["name"], c["H"], c["W"], c["T"], c["seed"])
    return P.write_pardom_scene(root, c["name"], c["H"], c["W"], c["T"], c["seed"], c["missing"])


def _mpl_imread(path):
    from PIL import Image
    with Image.open(path) as im:
        if im.mode in ("P", "LA"):
            im = im.convert("RGBA")
        assert im.mode in ("RGB", "RGBA"), (path, im.mode)
        return np.divide(np.asarray(im), 2 ** 8 - 1, dtype=np.float32)


class _Quaternion:
    def __init__(self, *q):
        self.q = q[0] if len(q) == 1 else q

    @property
    def rotation_matrix(self):
        return C.quaternion_rotation_matrix(self.q)


def _edit(code, edit):
    assert code.count(edit[0]) == 1, edit
    return code.replace(*edit)


def reference():
    """{kind: process_example} executed from the reference's data-gen sources."""
    import glob
    import time

    import PIL
    import PIL.Image  # noqa: F401
    if not ref_shim.available():
        raise RuntimeError("set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    dg = os.path.join(os.path.dirname(ref_shim.REF), "data-gen")
    noprint = lambda *a, **k: None
    uns = dict(np=np, json=__import__("json"), print=noprint)
    exec(compile(_cut(os.path.join(dg, "data_utils.py"), ["load_json", "camera_to_world", "unproject_pixels_to_points"]),
                 "data_utils.py", "exec"), uns)
    data_utils = types.SimpleNamespace(**{k: uns[k] for k in ("load_json", "camera_to_world", "unproject_pixels_to_points")})
    out = {}
    for kind, names in (("kubric", ["is_finished", "get_kubric_camera_matrices_torch", "correct_depth_ball_plane_torch",
                                    "process_example"]),
                        ("pardom", ["is_finished", "get_intrinsics_matrix", "get_extrinsics_matrix", "process_example"])):
        ns = dict(np=np, torch=torch, os=os, glob=glob, time=time, PIL=PIL, print=noprint, data_utils=data_utils,
                  tqdm=types.SimpleNamespace(tqdm=lambda x: x), plt=types.SimpleNamespace(imread=_mpl_imread),
                  Quaternion=_Quaternion, process_dtype=torch.float32, store_xyz_dtype=torch.float16, MAX_DEPTH=30000.0)
        exec(compile(_edit(_cut(os.path.join(dg, f"convert_pcl_{kind}.py"), names), DEVICE_EDIT), f"convert_pcl_{kind}.py",
                     "exec"), ns)
        out[kind] = ns["process_example"]
    return out


def oracle_frames(kind, scene, frames):
    """{t: the list the oracle stores} for frames t of a scene, read through gcd_b200.convert's readers (None: skipped frame)."""
    if kind == "kubric":
        cams, _ = C.kubric_cameras(scene, max(frames) + 1)
        paths = lambda t: C.kubric_frame_paths(scene, t)
    else:
        views = C.pardom_views(scene)
        cams = C.pardom_cameras(scene, views)
        paths = lambda t: C.pardom_frame_paths(scene, views, t)
    out = {}
    for t in frames:
        got = C.decode_frame(kind, paths(t))
        if got is None:
            out[t] = None
            continue
        depth, rgb, segm = got
        V = depth.shape[0]
        xyz = P.torch_chain(depth, cams[t] if kind == "kubric" else cams, kind)
        lst = [xyz, torch.from_numpy(rgb), torch.from_numpy(segm)]
        if kind == "pardom":
            lst.append(torch.arange(V, dtype=torch.uint8)[:, None, None].expand(V, rgb.shape[1], 1).contiguous())
        out[t] = lst
    return out


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.uint8) if a.dtype != torch.uint8 else a,
                                                                      b.view(torch.uint8) if b.dtype != torch.uint8 else b)


def main():
    ref = reference()
    with tempfile.TemporaryDirectory() as tmp:
        for c in (KUBRIC, PARDOM):
            scene = write_case(os.path.join(tmp, "data"), c)
            out_dir = os.path.join(tmp, "pcl", c["name"])
            frames = list(range(c["T"]))
            views = list(range(16 if c["kind"] == "kubric" else 19))
            ref[c["kind"]](0, 0, (scene, out_dir), views, frames, ["rgb", "segm"], 0, 0)
            stored = {}
            for t in frames:
                p = os.path.join(out_dir, C.output_name(c["kind"], t))
                stored[t] = torch.load(p, weights_only=True) if os.path.exists(p) else None
            mine = oracle_frames(c["kind"], scene, frames)
            for t in frames:
                assert (stored[t] is None) == (mine[t] is None), (c["name"], t)
                if stored[t] is not None:
                    assert len(stored[t]) == len(mine[t]) and all(same_bits(a, b) for a, b in zip(stored[t], mine[t])), (c["name"], t)
            meta = dict(reference=f"data-gen/convert_pcl_{c['kind']}.py process_example, data-gen/data_utils.py",
                        device_edit=DEVICE_EDIT,
                        replaced={"Quaternion(q).rotation_matrix": "gcd_b200.convert.quaternion_rotation_matrix (float64 restatement)",
                                  "plt.imread": "oracle.pin_convert._mpl_imread (np.divide(bytes, 255, dtype=float32); P, LA via RGBA)"},
                        torch=str(torch.__version__), numpy=np.__version__)
            path = os.path.join(GOLD, f"pcl_{c['kind']}.pt")
            torch.save({"meta": meta, "case": c, "frames": stored}, path)
            print(f"wrote {path} ({os.path.getsize(path)} bytes): frames {[t for t in frames if stored[t] is not None]} stored, "
                  f"oracle torch chain bit-identical")


if __name__ == "__main__":
    main()
