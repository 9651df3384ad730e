"""Host side of gcd_b200.evaluate against goldens written from the reference's own data modules (oracle/pin_evaluate.py):
trajectories, batch assembly and conditioning noise bit for bit, control rows of the shipped controls JSONs, the metrics-JSON key
set of scripts/test.py, the point-cloud readers, and the inputs that must raise."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from gcd_b200 import evaluate as E  # noqa: E402


def _gold(kind):
    return torch.load(os.path.join(GOLD, f"evaluate_{kind}.pt"), weights_only=False)


def _controls():
    with open(os.path.join(GOLD, "evaluate_controls.json")) as f:
        return json.load(f)


def _same(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    assert torch.equal(got, want), (what, (got.double() - want.double()).abs().max().item())


def _check_batch(kind, traj, case, gold):
    from oracle import pin_evaluate as P
    T = gold["meta"]["T"]
    for pi, (ti, to) in enumerate(gold["meta"]["padding"]):
        want = case[f"dict{pi}"]
        src, dst, rep = P.frames(case["_seed"] + pi)        # the frames and noise seed oracle/pin_evaluate.py used
        fps = int(want["fps_id"][0])
        cfg = gold["cfgs"][case["cfg"]]
        got = E.construct_batch(kind, traj, src, dst, rep, fps, torch.Generator().manual_seed(case["_seed"] + pi),
                                motion_bucket_range=cfg.get("motion_bucket_range"), input_frames=ti, output_frames=to)
        assert set(got) == set(want) - {"src_view_idx", "dst_view_idx"}
        for k in got:
            _same(got[k], want[k], f"{case['label']} cfg {case['cfg']} padding {pi}: {k}")
        assert got["cond_frames"].shape[0] == T


def _with_seeds(gold, base):
    for i, c in enumerate(gold["cases"]):
        c["_seed"] = base + 10 * i
    return gold["cases"]


def test_kubric_trajectories_and_batch_match_reference_bit_for_bit():
    gold = _gold("kubric")
    cases = _with_seeds(gold, 100)
    assert len(cases) == 15
    for case in cases:
        cfg = gold["cfgs"][case["cfg"]]
        row = case["row"].numpy()
        traj = E.kubric_trajectories(row, gold["meta"]["T"], cfg["trajectory"], cfg["move_time"], cfg["delta_azimuth_range"],
                                     cfg["delta_elevation_range"])
        for k in ("spherical_src", "spherical_dst", "extrinsics_src", "extrinsics_dst"):
            _same(traj[k], case[k], f"{case['label']} cfg {case['cfg']}: {k}")
        assert float(traj["motion_amount"]) == case["motion_amount"]
        _check_batch("kubric", traj, case, gold)


def test_pardom_trajectories_and_batch_match_reference_bit_for_bit():
    gold = _gold("pardom")
    cases = _with_seeds(gold, 500)
    assert len(cases) == 6
    for case in cases:
        cfg = gold["cfgs"][case["cfg"]]
        traj = E.pardom_trajectories(gold["intrinsics"].clone(), gold["meta"]["T"], trajectory=cfg["trajectory"],
                                     move_time=cfg["move_time"])
        for k in ("extrinsics_src", "extrinsics_dst", "intrinsics_src", "intrinsics_dst", "readable_angles"):
            _same(traj[k], case[k], f"{case['label']} cfg {case['cfg']}: {k}")
        assert traj["motion_amount"] == case["motion_amount"]
        _check_batch("pardom", traj, case, gold)


def test_control_rows_of_the_shipped_controls():
    from oracle import pin_evaluate as P
    fix = _controls()
    want = dict(P.kubric_rows(fix))
    for fn, scenes in fix["kubric"].items():
        for scene, samples in scenes.items():
            for sample, entry in samples.items():
                row = E.control_row("kubric", E.control_entry(scenes, f"/data/Kubric-4D/{scene}", int(sample[-2:])))
                assert row.dtype == np.float32 and np.array_equal(row, want[f"{fn}:{scene}:{sample}"])
                frames, fps = E.clip_frames("kubric", row)
                assert fps == entry["fps"] and frames[0] == entry["frame_start"] and frames[1] - frames[0] == entry["frame_skip"]
    a = P.EXPLICIT
    row = E.control_row("kubric", None, a["frame_start"], a["frame_stride"], a["frame_rate"], a["angles"])
    assert np.array_equal(row, want["explicit"])
    # command-line frame bounds override the entry's, angles always come from the entry (test.py:182-191)
    entry = fix["kubric"]["kubric_valtest_controls_gradual.json"]["scn02800"]["sample_00"]
    row = E.control_row("kubric", entry, frame_start=5, angles=(0, 0, 0, 0, 0, 0))
    assert row[0] == 5 and row[1] == entry["frame_skip"] and row[3] == np.float32(entry["spherical_start"][0])
    for fn, scenes in fix["pardom"].items():
        for scene, samples in scenes.items():
            for sample, entry in samples.items():
                row = E.control_row("pardom", entry)
                assert list(row[:3]) == [entry["frame_start"], entry["frame_skip"], entry["fps"]] and not row[3:].any()
                frames, fps = E.clip_frames("pardom", row)
                assert fps == entry["fps"] and len(frames) == 14


def test_metrics_json_keys_and_values_follow_test_py(tmp_path):
    keys = _gold("kubric")["metric_keys"]
    assert tuple(keys) == E.METRIC_KEYS + E.MASKED_METRIC_KEYS
    S, T = 2, 3
    m = {k: torch.rand(S, T, dtype=torch.float64) for k in keys if k.startswith("frame_") and "diversity" not in k}
    m.update({k: torch.rand(T, dtype=torch.float64) for k in keys if k.startswith("frame_diversity")})
    m.update({k: torch.rand(S, dtype=torch.float64) for k in keys if k.startswith("mean_") and "diversity" not in k})
    m.update({k: torch.rand((), dtype=torch.float64) for k in keys if k.startswith("mean_diversity")})
    m["frame_psnr_occ"][1, 2] = float("nan")
    m = dict(reversed(list(m.items())))
    p = tmp_path / "x" / "a_metrics.json"
    E.save_metrics_json(str(p), m)
    out = json.loads(p.read_text())
    assert list(out) == list(keys)
    assert isinstance(out["mean_diversity"], float) and len(out["frame_psnr"]) == S and len(out["frame_psnr"][0]) == T
    assert len(out["frame_diversity_vis"]) == T and len(out["mean_psnr_vis"]) == S
    assert math.isnan(out["frame_psnr_occ"][1][2]) and out["frame_ssim"][0][1] == m["frame_ssim"][0, 1].item()


def _write_kubric(d, frames, V=3, N=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    want = []
    for t in frames:
        x = (torch.randn(V, N, 3, generator=g) * 10).to(torch.float16)
        c = torch.randint(0, 256, (V, N, 3), generator=g, dtype=torch.uint8)
        torch.save([x, c, torch.zeros_like(c)], os.path.join(d, f"pcl_rgb_segm_{t:05d}.pt"))
        want.append((x, c))
    return want


def test_point_cloud_readers_round_trip(tmp_path):
    frames = [4, 6, 8]
    want = _write_kubric(str(tmp_path), frames)
    xyz, rgb = E.load_kubric_clouds(str(tmp_path), np.array(frames))
    assert xyz.dtype == torch.float16 and rgb.dtype == torch.uint8 and xyz.shape == (3, 3, 5, 3)
    for i, (x, c) in enumerate(want):
        assert torch.equal(xyz[i], x) and torch.equal(rgb[i], c)
    pd = tmp_path / "pardom"
    pd.mkdir()
    g = torch.Generator().manual_seed(1)
    stored = []
    for t in (0, 2):
        x = torch.randn(19, 4, 3, generator=g).to(torch.float16)
        x[0, 0, 0] = float("inf")                                   # ParDom clouds keep far points that overflow fp16
        c = torch.randint(0, 256, (19, 4, 3), generator=g, dtype=torch.uint8)
        s = torch.randint(0, 30, (19, 4, 1), generator=g, dtype=torch.uint8)
        torch.save([x, c, s, torch.zeros_like(s)], str(pd / f"pcl_rgb_segm_{t * 10 + 5:06d}.pt"))
        stored.append((x, c, s))
    xyz, rgb, segm = E.load_pardom_clouds(str(pd), [0, 2])
    for i, (x, c, s) in enumerate(stored):
        assert torch.equal(xyz[i], x) and torch.equal(rgb[i], c) and torch.equal(segm[i], s)


def test_scene_metadata_readers(tmp_path):
    scn = tmp_path / "scn00007"
    scn.mkdir()
    (scn / "scn00007_p0_v4.json").write_text(json.dumps({"camera": {"K": [[1.2, 0, -0.5], [0, -1.8, -0.5], [0, 0, -1]]}}))
    assert torch.equal(E.read_kubric_intrinsics(str(scn)), torch.tensor([[1.2, 0, 0.5], [0, 1.8, 0.5], [0, 0, 1]]))
    sc = tmp_path / "scene_000003" / "calibration"
    sc.mkdir(parents=True)
    names = ["yaw-0", "camera1", "velodyne", "camera0"]
    intr = [{"fx": 10.0 + i, "fy": 20.0 + i, "cx": 30.0, "cy": 40.0} for i in range(4)]
    (sc / "x.json").write_text(json.dumps({"names": names, "intrinsics": intr, "extrinsics": [{}] * 4}))
    K = E.read_pardom_intrinsics(str(tmp_path / "scene_000003"))
    assert K.shape == (3, 3, 3) and K[:, 0, 0].tolist() == [13.0, 11.0, 10.0]      # camera0, camera1, yaw-0


def test_random_branches_and_malformed_inputs_raise(tmp_path):
    with pytest.raises(NotImplementedError):
        E.kubric_trajectories(E.control_row("kubric", None, 0, 2, 12))            # no angles: range sampling
    K = torch.eye(3).repeat(19, 1, 1)
    for mode in (dict(input_mode="magic_random"), dict(output_mode="topdown2"), dict(input_mode="traffic1", output_mode="traffic1"),
                 dict(output_mode="magic_opposite")):
        with pytest.raises(NotImplementedError):
            E.pardom_trajectories(K, **mode)
    with pytest.raises(ValueError):
        E.pardom_trajectories(K, dst_azimuth_range=(-90.0, 90.0))
    with pytest.raises(ValueError):
        E.pardom_trajectories(K[:1])
    with pytest.raises(ValueError):
        E.kubric_trajectories(np.zeros(8, dtype=np.float32))
    with pytest.raises(ValueError):
        E.kubric_trajectories(np.zeros(9, dtype=np.float32), move_time=15)
    with pytest.raises(ValueError):
        E.kubric_trajectories(np.zeros(9, dtype=np.float32), trajectory="spline")
    with pytest.raises(ValueError):
        E.control_row("kubric")                                                     # no entry, no frame bounds
    with pytest.raises(ValueError):
        E.control_row("kubric", {"frame_start": 0, "frame_skip": 2})               # entry without angles
    with pytest.raises(ValueError):
        E.control_row("shapenet", None, 0, 1, 24)
    with pytest.raises(KeyError):
        E.control_entry({"scn00001": {"sample_00": {}}}, "/x/scn00001", 3)
    with pytest.raises(ValueError):
        E.clip_frames("kubric", E.control_row("kubric", None, 10, 4, 6, (0, 0, 0, 0, 15, 0)))   # frames 10..62 > 59
    with pytest.raises(ValueError):
        E.clip_frames("pardom", E.control_row("pardom", None, 0, 0, 10))
    traj = E.kubric_trajectories(E.control_row("kubric", None, 0, 2, 12, (0, 30, 10, 5, 15, 0)))
    f = torch.zeros(14, 3, 4, 6)
    with pytest.raises(ValueError):
        E.construct_batch("kubric", traj, f, torch.zeros(14, 3, 4, 8), None, 12, torch.Generator())
    with pytest.raises(ValueError):
        E.construct_batch("kubric", traj, f[:13], f[:13], None, 12, torch.Generator())
    # readers: missing file, wrong list length, wrong dtype, ragged frames
    with pytest.raises(FileNotFoundError):
        E.load_kubric_clouds(str(tmp_path), [0])
    torch.save([torch.zeros(2, 3, 3)], str(tmp_path / "pcl_rgb_segm_00000.pt"))
    with pytest.raises(ValueError):
        E.load_kubric_clouds(str(tmp_path), [0])
    torch.save([torch.zeros(2, 3, 3), torch.zeros(2, 3, 3), torch.zeros(2, 3, 3)], str(tmp_path / "pcl_rgb_segm_00000.pt"))
    with pytest.raises(ValueError):
        E.load_kubric_clouds(str(tmp_path), [0])
    _write_kubric(str(tmp_path), [0], N=5)
    _write_kubric(str(tmp_path), [1], N=6)
    with pytest.raises(ValueError):
        E.load_kubric_clouds(str(tmp_path), [0, 1])
    torch.save([torch.zeros(2, 3, 3, dtype=torch.float16), torch.zeros(2, 3, 3, dtype=torch.uint8),
                torch.zeros(2, 3, 3, dtype=torch.uint8), torch.zeros(2, 3, 1, dtype=torch.uint8)],
               str(tmp_path / "pcl_rgb_segm_000005.pt"))
    with pytest.raises(ValueError):
        E.load_pardom_clouds(str(tmp_path), [0])                                     # segm must be [V, N, 1]


def test_command_line_parses_and_needs_a_device(tmp_path):
    args = E.parser().parse_args(["--kind", "pardom", "--checkpoint", "x.ckpt", "--examples", "l.txt", "--pcl-root", "p",
                                  "--output", "o", "--num-samples", "3", "--motion-bucket-range", "127", "127"])
    assert args.num_samples == 3 and args.motion_bucket_range == [127, 127] and args.trajectory is None
    lst = tmp_path / "l.txt"
    lst.write_text("\n/datasets/Kubric-4D/data/scn02900\n# skipped\n/datasets/Kubric-4D/data/scn02901\n")
    assert E.read_examples(str(lst)) == ["/datasets/Kubric-4D/data/scn02900", "/datasets/Kubric-4D/data/scn02901"]
    s = E.summarize([{"mean_psnr": torch.tensor([20.0, 22.0])}, {"mean_psnr": torch.tensor([float("nan"), 30.0])}])
    assert s["examples"] == 2 and s["mean_psnr"] == 25.5
