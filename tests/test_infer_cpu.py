"""Host side of gcd_b200.infer against goldens written from the reference's own infer.py path (oracle/pin_infer.py): the crop
box, the float64 frame oracle against the reference's frames and against cv2, the custom-clip batch bit for bit, input
discovery, output names, the sample spread, and the command line's early refusals. No GPU."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from gcd_b200 import infer as I  # noqa: E402
from oracle import frames_oracle as F, pin_infer as P  # noqa: E402

TOL = 2.4e-7     # two fp32 ulps at 1.0


def _gold(name):
    return torch.load(os.path.join(GOLD, f"infer_{name}.pt"), weights_only=False)


def test_crop_box_matches_center_crop_numpy():
    crops = _gold("frames")["crops"]
    assert len(crops) == len(P.CROP_CASES)
    for c in crops:
        assert I.crop_box(c["H"], c["W"], c["frame_hw"]) == tuple(c["box"]), c
        assert I.crop_box(c["H"], c["W"], c["frame_hw"], center_crop=False) == (0, 0, c["H"], c["W"])


def _cases():
    g = _gold("frames")
    for c in g["images"]:
        yield c, P.seeded_frames(c["shape"], c["seed"])[None], c["input_rgb"][None]
    for c in g["videos"]:
        yield c, P.seeded_frames(c["shape"], c["seed"])[list(c["frames"])], c["input_rgb"]


def test_frames_oracle_matches_reference_frames():
    n = 0
    for c, u8, want in _cases():
        got = torch.from_numpy(F.prepare(u8, c["frame_hw"], bool(c["center_crop"])))
        assert got.shape == want.shape and got.dtype == want.dtype
        err = (got.double() - want.double()).abs().max().item()
        print(f"{tuple(u8.shape)} -> {c['frame_hw']} crop {c['center_crop']}: max |oracle - reference| {err:.2e}")
        assert err <= TOL
        if tuple(c["shape"][:2]) == tuple(c["frame_hw"]) or I.crop_box(*c["shape"][:2], c["frame_hw"])[2:] == tuple(c["frame_hw"]):
            assert torch.equal(got, want)                     # no resize: exact
        n += 1
    assert n == len(P.IMAGE_CASES) + len(P.VIDEO_CASES)


def test_frames_oracle_round_trip_is_not_the_identity():
    p = np.float32(np.arange(256) / np.float32(255))
    assert (F.round_trip(p) != p).any() and (F.round_trip(p)[p >= 0.5] == p[p >= 0.5]).all()


def test_frames_oracle_within_two_ulp_of_cv2():
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)          # OpenCV's generic INTER_LINEAR path (IPP builds differ by up to 4e-5 at some ratios)
    try:
        rng = np.random.default_rng(3)
        for H, W, h, w in ((426, 640, 256, 384), (200, 300, 256, 384), (1080, 1620, 576, 864), (720, 1280, 256, 384),
                           (128, 192, 64, 96), (90, 70, 64, 128)):
            img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8).astype(np.float32) / np.float32(255)
            ref = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
            err = np.abs(F.resize_linear(img, (h, w)).astype(np.float64) - ref).max()
            print(f"{H}x{W} -> {h}x{w}: max |oracle - cv2| {err:.2e}")
            assert err <= TOL
    finally:
        cv2.ipp.setUseIPP(ipp)


def test_construct_batch_matches_reference_bit_for_bit():
    g = _gold("host")
    assert len(g["batches"]) == len(P.BUNDLES) * len(P.CONTROLS)
    for case in g["batches"]:
        label, az, el, traj, mt, cam, mbr = g["bundles"][case["bundle"]]
        da, de, dr, fr, mid, ca, force = g["controls"][case["controls"]]
        kind = "kubric" if cam == "spherical" else "pardom"
        got = I.construct_batch(kind, P.seeded_input(case["seed"]), da, de, dr, fr, mid, ca,
                                torch.Generator().manual_seed(case["seed"]), bool(force), traj, mt, az, el, mbr)
        want = case["batch"]
        assert list(got) == list(want), (label, list(got), list(want))
        for k, v in want.items():
            if torch.is_tensor(v):
                assert got[k].dtype == v.dtype and got[k].shape == v.shape and torch.equal(got[k], v), (label, case["controls"], k)
            else:
                assert got[k] == v, (label, k)


def test_input_discovery_matches_reference(tmp_path, monkeypatch):
    g = _gold("host")
    P.make_tree(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    assert len(g["discovery"]) == len(P.DISCOVERY)
    for paths, want in g["discovery"]:
        assert I.list_inputs(paths) == want, paths


def test_output_names_match_reference():
    for output, index, example, ckpt, model, prefix in _gold("host")["names"]:
        assert I.model_name(ckpt) == model
        assert I.output_stem(output, index, example, model) == prefix


def test_sample_diversity_matches_infer_calculate_metrics():
    from gcd_b200 import metrics
    want = _gold("host")["diversity"]
    unc, fd, md = metrics.sample_diversity(P.seeded_samples())
    assert unc.shape == want["uncertainty"].shape and fd.shape == want["frame_diversity"].shape
    assert (unc - want["uncertainty"]).abs().max().item() < 1e-6
    assert (fd - want["frame_diversity"].double()).abs().max().item() < 1e-6
    assert abs(md.item() - want["mean_diversity"]) < 1e-6
    _, fd1, md1 = metrics.sample_diversity(P.seeded_samples(S=1))
    assert md1.item() == 0.0 and (fd1 == 0).all()


def test_readers_refuse_what_they_cannot_read(tmp_path):
    from torchvision.io import write_png
    gray = tmp_path / "gray.png"
    write_png(torch.zeros(1, 8, 8, dtype=torch.uint8), str(gray))
    with pytest.raises(ValueError, match="grayscale"):
        I.read_frames(str(gray), [0])
    folder = tmp_path / "frames"
    folder.mkdir()
    for t in range(3):
        write_png(torch.full((3, 8, 8), t, dtype=torch.uint8), str(folder / f"{t:04d}.png"))
    imgs, cmap = I.read_frames(str(folder), [0, 2])
    assert cmap == (0, 1, 2) and [int(x[0, 0, 0]) for x in imgs] == [0, 2]
    with pytest.raises(ValueError, match="run past"):
        I.read_frames(str(folder), [1, 3])
    still, _ = I.read_frames(str(folder / "0001.png"), I.clip_frames(4, 0, 2))
    assert len(still) == 4 and all(x is still[0] for x in still)
    with pytest.raises(ValueError, match="8-bit"):
        I._check_u8(torch.zeros(3, 4, 4, dtype=torch.uint16), "deep.png")


def test_video_reader_decodes_only_the_clip_and_refuses_frames_past_the_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    path = str(tmp_path / "clip.mp4")
    w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 8.0, (64, 32))
    assert w.isOpened()
    for t in range(5):
        w.write(np.full((32, 64, 3), 40 * t, dtype=np.uint8))
    w.release()
    frames = I.read_video(path, [1, 3])
    assert frames.shape == (2, 32, 64, 3) and frames.dtype == torch.uint8
    assert abs(int(frames[1].double().mean()) - 120) <= 3
    with pytest.raises(ValueError, match="run past"):
        I.read_video(path, [2, 5])


def test_command_line_refuses_bad_resolution_and_mp4_without_cv2(tmp_path, monkeypatch, capsys):
    base = ["--kind", "kubric", "--checkpoint", "x.ckpt", "--input", str(tmp_path), "--output", str(tmp_path / "out")]
    for bad in (["--frame-width", "380"], ["--frame-height", "0"]):
        with pytest.raises(SystemExit):
            I.main(base + bad)
        assert "multiple of 64" in capsys.readouterr().err
    monkeypatch.setitem(sys.modules, "cv2", None)          # `import cv2` raises ImportError
    with pytest.raises(SystemExit, match="needs OpenCV"):
        I.main(base + ["--save-mp4", "1"])
    assert not (tmp_path / "out").exists()
