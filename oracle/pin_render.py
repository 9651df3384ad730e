"""Writes tests/golden/render_{kubric,pardom}.pt from the reference's own renderer (needs a reference checkout: GCD_REFERENCE, see
oracle/ref_shim.py) and asserts oracle/render_oracle.py against it.

    python -m oracle.pin_render

`world_to_camera`, `project_points_to_pixels`, `spreaded_index_add`, `gaussian_blur_masked_vectorized` and `blur_into_black` are cut
out of gcd-model/sgm/data/geometry.py with `ast`, and `synth_src_dst_rgb` / `synth_rgb` out of kubric_arbit.py / pardom_arbit.py.
geometry.py itself cannot be imported here (cv2, lovely_tensors, mediapy, ...), the cut functions run with the real torch,
torchvision and einops on CPU over a stub `self` and a no-op `print`. The one edit to the executed source is the hard-coded
`device = f'cuda:{self.data_gpu}'`, which becomes `device = 'cpu'` (recorded in the goldens' metadata).

Clouds and cameras are regenerated from seeds (render_oracle.synthetic_clouds); only the reference outputs are stored.
"""
import ast
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from oracle import render_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
DEVICE_EDIT = ("device = f'cuda:{self.data_gpu}'", "device = 'cpu'")
RENDER_HW, FRAME_HW = (56, 84), (48, 72)

# golden cases: the clouds and trajectories the tests regenerate
KUBRIC = dict(kind="kubric", T=3, V=16, h=24, w=36, seed=11, src=(10.0, 40.0, 14.0, 3.0), dst=(95.0, 140.0, 13.0, 4.0))
PARDOM = dict(kind="pardom", T=3, V=19, h=24, w=32, seed=12, traj=((16 / 19) * 360.0 - 8.0, (16 / 19) * 360.0 + 8.0, 14.0, 3.0))


def kubric_case(c=KUBRIC):
    cl = O.synthetic_clouds(c["kind"], c["T"], c["V"], c["h"], c["w"], c["seed"])
    return cl, O.trajectory(c["T"], *c["src"]), O.trajectory(c["T"], *c["dst"])


def pardom_case(c=PARDOM):
    cl = O.synthetic_clouds(c["kind"], c["T"], c["V"], c["h"], c["w"], c["seed"])
    return cl, O.trajectory(c["T"], *c["traj"])


def _cut(path, names, cls=None, edit=None):
    src = open(path).read()
    tree = ast.parse(src)
    nodes = tree.body
    if cls is not None:
        nodes = next(n for n in nodes if isinstance(n, ast.ClassDef) and n.name == cls).body
    body = [n for n in nodes if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), (path, names)
    code = "\n\n".join(ast.get_source_segment(src, n) for n in body)
    import textwrap
    code = textwrap.dedent(code)
    if edit is not None:
        assert code.count(edit[0]) == 1, edit
        code = code.replace(*edit)
    return code


def reference():
    """Returns (geometry namespace, synth_src_dst_rgb, synth_rgb) executed from the reference's source."""
    import numpy as np
    import torchvision
    from einops import rearrange
    if not ref_shim.available():
        raise RuntimeError("set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    data = os.path.join(ref_shim.REF, "sgm", "data")
    noprint = lambda *a, **k: None
    gns = dict(torch=torch, torchvision=torchvision, rearrange=rearrange, np=np, time=__import__("time"), print=noprint)
    exec(compile(_cut(os.path.join(data, "geometry.py"), ["world_to_camera", "project_points_to_pixels", "spreaded_index_add",
                                                          "gaussian_blur_masked_vectorized", "blur_into_black"]),
                 "geometry.py", "exec"), gns)
    geometry = types.SimpleNamespace(**{k: gns[k] for k in ("world_to_camera", "project_points_to_pixels", "spreaded_index_add",
                                                           "gaussian_blur_masked_vectorized", "blur_into_black")})
    ns = dict(torch=torch, geometry=geometry, rearrange=rearrange, np=np, print=noprint)
    exec(compile(_cut(os.path.join(data, "kubric_arbit.py"), ["synth_src_dst_rgb"], "KubricSynthViewDataset", DEVICE_EDIT),
                 "kubric_arbit.py", "exec"), ns)
    exec(compile(_cut(os.path.join(data, "pardom_arbit.py"), ["synth_rgb"], "ParallelDomainSynthViewDataset", DEVICE_EDIT),
                 "pardom_arbit.py", "exec"), ns)
    return geometry, ns["synth_src_dst_rgb"], ns["synth_rgb"]


def stub_self(T, reproject, modal_time=0, palette=None):
    return types.SimpleNamespace(model_frames=T, render_height=RENDER_HW[0], render_width=RENDER_HW[1], frame_height=FRAME_HW[0],
                                 frame_width=FRAME_HW[1], spread_radius=1, reproject_rgbd=reproject, data_gpu=0,
                                 modal_time=modal_time, ontology={"semantic_id_rgb_map": palette})


def run_kubric(synth, cl, src, dst):
    T = cl["xyz"].shape[0]
    pcl = {"xyz": list(cl["xyz"]), "rgb": list(cl["rgb"]), "segm_rgb": None}
    intr = cl["intrinsics"]
    return synth(stub_self(T, True), pcl, src, dst, intr, src)


def run_pardom(synth, cl, ext, modality, modal_time, reproject):
    T = cl["xyz"].shape[0]
    pcl = {"xyz": list(cl["xyz"]), "rgb": list(cl["rgb"]), "segm": list(cl["segm"]), "tag": None}
    return synth(stub_self(T, reproject, modal_time, cl["palette"]), pcl, modality, ext, cl["intrinsics"], reproject)


def edge_cloud():
    """Points behind / too near the camera, uv in (-1.5, -0.5), non-finite fp16 coordinates, a Kubric-range scene (max depth < 64)."""
    RT = torch.eye(4, dtype=torch.float32)
    K = torch.tensor([[40.0, 0, 20.0], [0, 40.0, 15.0], [0, 0, 1]])
    H, W = 30, 40
    g = torch.Generator().manual_seed(3)
    n = 4000
    z = 2 + 10 * torch.rand(n, generator=g, dtype=torch.float64)
    u = -2 + (W + 4) * torch.rand(n, generator=g, dtype=torch.float64)
    v = -2 + (H + 4) * torch.rand(n, generator=g, dtype=torch.float64)
    u[:200] = -1.5 + torch.rand(200, generator=g, dtype=torch.float64)       # (-1.5, -0.5) -> column 0 by truncation
    v[200:400] = -1.5 + torch.rand(200, generator=g, dtype=torch.float64)
    z[400:500] = 0.05                                                         # depth <= 0.1
    z[500:600] = -3.0                                                         # behind the camera
    xyz = torch.stack([(u - 20) * z / 40, (v - 15) * z / 40, z], -1).to(torch.float16)
    xyz[600:650, 2] = float("inf")
    xyz[650:700, 0] = float("-inf")
    xyz[700:720] = float("nan")
    rgb = torch.randint(0, 256, (n, 3), generator=g, dtype=torch.uint8)
    return xyz, rgb, K, RT, (H, W)


def main():
    geometry, synth_k, synth_p = reference()
    meta = {"source": "gcd-model/sgm/data/{geometry,kubric_arbit,pardom_arbit}.py, cut with ast and run on CPU",
            "edit": f"{DEVICE_EDIT[0]!r} -> {DEVICE_EDIT[1]!r}", "render_hw": RENDER_HW, "frame_hw": FRAME_HW}

    def agree(a, b, what):
        d = (a - b).abs().max().item()
        print(f"  oracle vs reference {what}: max-abs {d:.2e}")
        assert d < 1e-5, (what, d)

    # the oracle against the reference's own functions on the edge cloud, both strength branches
    xyz, rgb, K, RT, (H, W) = edge_cloud()
    for scale in (1.0, 8.0):
        x = (xyz.float() * scale).to(torch.float16)
        xr = torch.cat([x.double(), (rgb / 255.0).double()], 1)
        ref = geometry.project_points_to_pixels(xr, K, RT, H, W, spread_radius=1)[0]
        agree(O.project(x.float(), (rgb / 255.0).float(), K, RT, H, W, 1), ref, f"project x{scale}")
        for k in (21, 3):
            agree(O.blur_into_black(ref, k, k / 4.0), geometry.blur_into_black(ref, kernel_size=k, sigma=k / 4.0), f"blur k={k}")
    for rad in (1, 2, 3):
        t = torch.zeros(H * W, 1, dtype=torch.float64)
        t2 = t.clone()
        inds = torch.arange(0, H * W, 37)
        vals = torch.rand(len(inds), 1, dtype=torch.float64)
        geometry.spreaded_index_add(t, inds, vals, H, W, rad)
        O._index_add_spread(t2, inds, vals, H, W, rad)
        assert torch.equal(t, t2), rad

    cl, src, dst = kubric_case()
    s, d, r = run_kubric(synth_k, cl, src, dst)
    os_, od, orp = O.kubric_views(cl["xyz"], cl["rgb"], cl["intrinsics"][0], src, dst, True, RENDER_HW, FRAME_HW)
    for a, b, w in ((os_, s, "kubric src"), (od, d, "kubric dst"), (orp, r, "kubric reproject")):
        agree(a, b.float(), w)
    torch.save(dict(meta=meta, case=KUBRIC, rgb_src=s.float(), rgb_dst=d.float(), reproject=r.float()),
               os.path.join(GOLD, "render_kubric.pt"))

    cl, ext = pardom_case()
    out = dict(meta=meta, case=PARDOM)
    for name, modality, mt, rep in (("rgb", "rgb", 0, True), ("segm0", "segm", 0, False), ("segm2", "segm", 2, True)):
        o, rp = run_pardom(synth_p, cl, ext, modality, mt, rep)
        oo, orp = O.pardom_views(cl["xyz"], cl["rgb"], cl["intrinsics"], ext, modality, cl["segm"], cl["palette"], mt, rep,
                                 RENDER_HW, FRAME_HW)
        agree(oo, o.float(), f"pardom {name}")
        out[name] = o.float()
        if rep:
            agree(orp, rp.float(), f"pardom {name} reproject")
            out[name + "_reproject"] = rp.float()
    torch.save(out, os.path.join(GOLD, "render_pardom.pt"))
    for f in ("render_kubric.pt", "render_pardom.pt"):
        print(f, os.path.getsize(os.path.join(GOLD, f)))


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
