"""Writes tests/golden/evaluate_{kubric,pardom}.pt and tests/golden/evaluate_controls.json from the reference's own data modules
(needs a reference checkout: GCD_REFERENCE, see oracle/ref_shim.py).

    python -m oracle.pin_evaluate

`sample_trajectories` and `construct_dict` are cut out of gcd-model/sgm/data/kubric_arbit.py and pardom_arbit.py with `ast`,
`construct_trajectory` out of common.py and `cartesian_from_spherical` / `extrinsics_from_look_at` out of geometry.py (neither
module imports here: cv2, mediapy, pyquaternion, lovely_tensors, ...). They run on CPU over a stub `self` and a no-op `print`,
without edits, for a few control rows of eval/list/*_valtest_controls*.json (copied to evaluate_controls.json) and the
trajectory settings of the shipped configs (pretrained/*.yaml). The conditioning noise is the global CPU generator's after
`torch.manual_seed(seed)`; frames are regenerated from seeds, only the reference's outputs are stored. The metrics keys of
scripts/test.py (`metrics_dict['...']`, :474-494) are read from its source and stored too.
"""
import ast
import json
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
T, FH, FW = 14, 4, 6
# (controls file, scene, sample) rows copied into the fixture
KUBRIC_ROWS = (("kubric_valtest_controls_gradual.json", "scn02800", "sample_00"),
               ("kubric_valtest_controls_gradual.json", "scn02801", "sample_03"),
               ("kubric_valtest_controls_jumpy.json", "scn02900", "sample_01"),
               ("kubric_valtest_controls_jumpy.json", "scn02905", "sample_03"))
PARDOM_ROWS = (("pardom_valtest_controls.json", "scene_000000", "sample_00"),
               ("pardom_valtest_controls.json", "scene_000048", "sample_01"))
# test.py's default explicit angles (--azimuth_start 20 --delta_azimuth 30 --elevation_start 10 --delta_elevation 15
# --radius_start 15 --delta_radius 0) with frame bounds given on the command line
EXPLICIT = dict(angles=(20.0, 30.0, 10.0, 15.0, 15.0, 0.0), frame_start=3, frame_stride=2, frame_rate=12)
# trajectory settings of the shipped configs: gradual / direct, max 180 / max 90 (pretrained/kubric_*.yaml), one sine variant
KUBRIC_CFGS = (dict(trajectory="interpol_linear", move_time=13, delta_azimuth_range=[-180.0, 180.0],
                    delta_elevation_range=[-60.0, 60.0], motion_bucket_range=[0, 255]),
               dict(trajectory="interpol_linear", move_time=0, delta_azimuth_range=[-90.0, 90.0],
                    delta_elevation_range=[-30.0, 30.0], motion_bucket_range=[0, 255]),
               dict(trajectory="interpol_sine", move_time=7, delta_azimuth_range=[-90.0, 90.0],
                    delta_elevation_range=[-30.0, 30.0], motion_bucket_range=[127, 127]))
PARDOM_CFGS = (dict(trajectory="interpol_sine", move_time=13), dict(trajectory="interpol_sine", move_time=0),
               dict(trajectory="interpol_linear", move_time=5))
# construct_dict padding cases: (input_frames, output_frames)
PADDING = ((14, 14), (7, 10))


def _cut(path, names, cls=None):
    src = open(path).read()
    nodes = ast.parse(src).body
    if cls is not None:
        nodes = next(n for n in nodes if isinstance(n, ast.ClassDef) and n.name == cls).body
    body = [n for n in nodes if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), (path, names)
    return textwrap.dedent("\n\n".join(ast.get_source_segment(src, n) for n in body))


def reference():
    """Returns a namespace of the reference's functions, executed from its source."""
    if not ref_shim.available():
        raise RuntimeError("set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    data = os.path.join(ref_shim.REF, "sgm", "data")
    noprint = lambda *a, **k: None
    gns = dict(np=np, torch=torch, print=noprint)
    exec(compile(_cut(os.path.join(data, "geometry.py"), ["cartesian_from_spherical", "extrinsics_from_look_at"]),
                 "geometry.py", "exec"), gns)
    exec(compile(_cut(os.path.join(data, "common.py"), ["construct_trajectory"]), "common.py", "exec"), gns)
    geometry = types.SimpleNamespace(cartesian_from_spherical=gns["cartesian_from_spherical"],
                                     extrinsics_from_look_at=gns["extrinsics_from_look_at"])
    common = types.SimpleNamespace(construct_trajectory=gns["construct_trajectory"])
    out = {}
    for mod, cls in (("kubric_arbit", "KubricSynthViewDataset"), ("pardom_arbit", "ParallelDomainSynthViewDataset")):
        ns = dict(np=np, torch=torch, geometry=geometry, common=common, print=noprint)
        exec(compile(_cut(os.path.join(data, mod + ".py"), ["sample_trajectories", "construct_dict"], cls), mod + ".py", "exec"), ns)
        out[mod] = (ns["sample_trajectories"], ns["construct_dict"])
    return out


def metric_keys():
    """The keys scripts/test.py assigns into `metrics_dict`, in source order."""
    src = open(os.path.join(ref_shim.REF, "scripts", "test.py")).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "calculate_metrics")
    keys = []
    for n in ast.walk(fn):
        if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Subscript):
            t = n.targets[0]
            if isinstance(t.value, ast.Name) and t.value.id == "metrics_dict":
                keys.append(t.slice.value)
    return sorted(set(keys), key=keys.index)


def fixture():
    """A handful of rows of the controls JSONs (each full file is MBs)."""
    lst = os.path.join(os.path.dirname(ref_shim.REF), "eval", "list")
    out = {"kubric": {}, "pardom": {}}
    for kind, rows in (("kubric", KUBRIC_ROWS), ("pardom", PARDOM_ROWS)):
        cache = {}
        for fn, scene, sample in rows:
            if fn not in cache:
                with open(os.path.join(lst, fn)) as f:
                    cache[fn] = json.load(f)
            out[kind].setdefault(fn, {}).setdefault(scene, {})[sample] = cache[fn][scene][sample]
    return out


def frames(seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(T, 3, FH, FW, generator=g) * 2 - 1 for _ in range(3)]


def pardom_intrinsics(seed=5):
    """Pixel intrinsics [19, 3, 3] float32 of a ParDom-like rig (16 magic + 3 ego cameras)."""
    g = torch.Generator().manual_seed(seed)
    K = torch.zeros(19, 3, 3, dtype=torch.float32)
    K[:, 0, 0] = 400 + 200 * torch.rand(19, generator=g)
    K[:, 1, 1] = K[:, 0, 0] * (1 + 0.01 * torch.rand(19, generator=g))
    K[:, 0, 2] = 320 + torch.rand(19, generator=g)
    K[:, 1, 2] = 240 + torch.rand(19, generator=g)
    K[:, 2, 2] = 1.0
    return K


def kubric_rows(fix):
    """(label, row float32 [9]) of the fixture's Kubric entries (test.py:182-191) and of the explicit angles (:137-141)."""
    rows = []
    for fn, scenes in fix["kubric"].items():
        for scene, samples in scenes.items():
            for sample, e in samples.items():
                r = np.array([e["frame_start"], e["frame_skip"], 0, e["spherical_start"][0], e["spherical_end"][0],
                              e["spherical_start"][1], e["spherical_end"][1], e["spherical_start"][2], e["spherical_end"][2]],
                             dtype=np.float32)
                r[2] = int(round(24 / r[1]))
                rows.append((f"{fn}:{scene}:{sample}", r))
    a0, da, e0, de, r0, dr = EXPLICIT["angles"]
    rows.append(("explicit", np.array([EXPLICIT["frame_start"], EXPLICIT["frame_stride"], EXPLICIT["frame_rate"], a0, a0 + da, e0,
                                       e0 + de, r0, r0 + dr], dtype=np.float32)))
    return rows


def main():
    ref = reference()
    fix = fixture()
    with open(os.path.join(GOLD, "evaluate_controls.json"), "w") as f:
        json.dump(fix, f, indent=1)
    keys = metric_keys()
    meta = {"source": "gcd-model/sgm/data/{kubric_arbit,pardom_arbit,common,geometry}.py, cut with ast and run on CPU unedited",
            "T": T, "frame_hw": (FH, FW), "padding": PADDING}

    traj_k, dict_k = ref["kubric_arbit"]
    cases = []
    for label, row in kubric_rows(fix):
        for ci, cfg in enumerate(KUBRIC_CFGS):
            me = types.SimpleNamespace(model_frames=T, input_frames=T, output_frames=T, input_mode="arbitrary",
                                       output_mode="arbitrary", next_example=[0, int(row[1]), int(row[0]), False, *row[3:9]],
                                       cond_aug=0.02, frame_height=FH, frame_width=FW, **cfg)
            _, _, s_src, s_dst, e_src, e_dst, motion = traj_k(me, False)
            case = dict(label=label, row=torch.from_numpy(row), cfg=ci, spherical_src=s_src, spherical_dst=s_dst,
                        extrinsics_src=e_src, extrinsics_dst=e_dst, motion_amount=float(motion))
            fps = int(round(24 / int(row[1])))
            for pi, (ti, to) in enumerate(PADDING):
                me.input_frames, me.output_frames = ti, to
                seed = 100 + 10 * len(cases) + pi
                src, dst, rep = frames(seed)
                torch.manual_seed(seed)
                case[f"dict{pi}"] = dict_k(me, src, dst, rep, fps, s_src, s_dst, e_src, e_dst, motion, False)
            cases.append(case)
    torch.save(dict(meta=meta, cfgs=KUBRIC_CFGS, metric_keys=keys, cases=cases), os.path.join(GOLD, "evaluate_kubric.pt"))

    traj_p, dict_p = ref["pardom_arbit"]
    K = pardom_intrinsics()
    cases = []
    for fn, scenes in fix["pardom"].items():
        for scene, samples in scenes.items():
            for sample, e in samples.items():
                for ci, cfg in enumerate(PARDOM_CFGS):
                    me = types.SimpleNamespace(model_frames=T, input_frames=T, output_frames=T, input_mode="ego_forward",
                                               output_mode="topdown1", next_example=[0, scene, e["frame_skip"], e["frame_start"],
                                                                                     False],
                                               dst_cam_position=[-8.0, 0.0, 8.0], dst_cam_look_at=[5.6, 0.0, 1.55],
                                               dst_azimuth_range=[0.0, 0.0], cond_aug=0.02, motion_bucket_range=[127, 127],
                                               frame_height=FH, frame_width=FW, **cfg)
                    e_src, e_dst, k_src, k_dst, angles, sv, dv, motion = traj_p(me, torch.eye(4).repeat(19, 1, 1), K.clone(), False)
                    case = dict(label=f"{fn}:{scene}:{sample}", cfg=ci, extrinsics_src=e_src, extrinsics_dst=e_dst,
                                intrinsics_src=k_src, intrinsics_dst=k_dst, readable_angles=angles, motion_amount=float(motion))
                    fps = int(round(10 / int(e["frame_skip"])))
                    for pi, (ti, to) in enumerate(PADDING):
                        me.input_frames, me.output_frames = ti, to
                        seed = 500 + 10 * len(cases) + pi
                        src, dst, rep = frames(seed)
                        torch.manual_seed(seed)
                        case[f"dict{pi}"] = dict_p(me, src, dst, rep, fps, angles, sv, dv, e_src, e_dst, k_src, k_dst, motion,
                                                   False)
                    cases.append(case)
    torch.save(dict(meta=meta, cfgs=PARDOM_CFGS, intrinsics=K, cases=cases), os.path.join(GOLD, "evaluate_pardom.pt"))
    for f in ("evaluate_kubric.pt", "evaluate_pardom.pt", "evaluate_controls.json"):
        print(f, os.path.getsize(os.path.join(GOLD, f)))
    print("test.py metrics keys:", keys)


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
