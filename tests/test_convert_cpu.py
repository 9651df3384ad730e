"""gcd_b200.convert's host side on the CPU: the reference's stored lists (tests/golden/pcl_*.pt, oracle/pin_convert.py) against the
oracle's torch chain over the same regenerated scenes, the uint8 identity the colour planes rest on, the readers and their refusals,
the camera restatements, scene discovery, the skip rule, atomic writes and the command line's refusals."""
import io
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from gcd_b200 import convert as C  # noqa: E402


@pytest.mark.parametrize("kind", ["kubric", "pardom"])
def test_goldens_vs_oracle(kind, tmp_path):
    from oracle import pin_convert as PC
    g = torch.load(os.path.join(GOLD, f"pcl_{kind}.pt"), weights_only=True)
    scene = PC.write_case(str(tmp_path), g["case"])
    mine = PC.oracle_frames(kind, scene, sorted(g["frames"]))
    for t, want in g["frames"].items():
        if want is None:
            assert kind == "pardom" and mine[t] is None and t == g["case"]["missing"][0]
            continue
        assert len(mine[t]) == len(want) == (3 if kind == "kubric" else 4)
        for a, b in zip(mine[t], want):
            assert PC.same_bits(a, b), (kind, t)


def test_uint8_identity():
    v = np.arange(256)
    f = np.divide(v.astype(np.uint8), 255, dtype=np.float32)
    assert (f * np.float32(255.0)).astype(np.uint8).tolist() == v.tolist()
    t = (torch.from_numpy(f) * 255.0).type(torch.uint8)
    assert t.tolist() == v.tolist()


def _png_bytes(a, mode, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(a, mode).save(b, "PNG", **kw)
    return b.getvalue()


def test_png_modes(tmp_path):
    from PIL import Image
    rng = np.random.default_rng(0)
    rgba = rng.integers(0, 256, (5, 7, 4), dtype=np.uint8)
    for mode, arr in (("RGBA", rgba), ("RGB", rgba[..., :3].copy())):
        p = tmp_path / f"{mode}.png"
        p.write_bytes(_png_bytes(arr, mode))
        assert np.array_equal(C.read_png(str(p), 3), rgba[..., :3])
        assert np.array_equal(C.read_png(str(p), 1), rgba[..., 0])
    idx = rng.integers(0, 4, (5, 7), dtype=np.uint8)
    im = Image.fromarray(idx, "P")
    pal = np.array([[10, 20, 30], [40, 50, 60], [70, 80, 90], [200, 210, 220]], np.uint8)
    im.putpalette(pal.reshape(-1).tolist())
    im.save(tmp_path / "p.png")
    assert np.array_equal(C.read_png(str(tmp_path / "p.png"), 3), pal[idx])
    la = rng.integers(0, 256, (5, 7, 2), dtype=np.uint8)
    Image.fromarray(la, "LA").save(tmp_path / "la.png")
    assert np.array_equal(C.read_png(str(tmp_path / "la.png"), 3), np.repeat(la[..., :1], 3, -1))


def test_png_refusals(tmp_path):
    from PIL import Image
    p = tmp_path / "grey.png"
    Image.fromarray(np.zeros((4, 4), np.uint8), "L").save(p)
    with pytest.raises(ValueError, match="grey.png: greyscale"):
        C.read_png(str(p), 3)
    p16 = tmp_path / "deep.png"
    Image.fromarray(np.zeros((4, 4), np.uint16), "I;16").save(p16)
    with pytest.raises(ValueError, match="deep.png: 16-bit"):
        C.read_png(str(p16), 1)
    bad = tmp_path / "x.png"
    bad.write_bytes(b"not a png at all, not at all")
    with pytest.raises(ValueError, match="x.png: not a PNG"):
        C.read_png(str(bad), 3)


def test_depth_readers(tmp_path):
    from PIL import Image
    d = np.arange(12, dtype=np.float32).reshape(3, 4) - 2.5
    Image.fromarray(d, "F").save(tmp_path / "d.tiff")
    assert np.array_equal(C.read_tiff_depth(str(tmp_path / "d.tiff")), d)
    np.savez(tmp_path / "d.npz", data=d.astype(np.float64).reshape(3, 4, 1))
    got = C.read_npz_depth(str(tmp_path / "d.npz"), 3, 4)
    assert got.dtype == np.float32 and np.array_equal(got, d)
    with pytest.raises(ValueError, match="d.npz: depth holds 12 values"):
        C.read_npz_depth(str(tmp_path / "d.npz"), 4, 4)
    np.savez(tmp_path / "e.npz", other=d)
    with pytest.raises(ValueError, match="e.npz: no 'data'"):
        C.read_npz_depth(str(tmp_path / "e.npz"), 3, 4)


def test_quaternion_restatement():
    assert np.array_equal(C.quaternion_rotation_matrix([1, 0, 0, 0]), np.eye(3))
    s = np.sqrt(0.5)
    rz = C.quaternion_rotation_matrix([s, 0, 0, s])          # +90 degrees about z
    assert np.allclose(rz, [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-15)
    rx = C.quaternion_rotation_matrix([0, 1, 0, 0])          # 180 degrees about x
    assert np.allclose(rx, np.diag([1.0, -1.0, -1.0]), atol=1e-15)
    q = np.array([0.3, -1.2, 0.7, 2.0])
    r = C.quaternion_rotation_matrix(q)
    assert np.array_equal(r, C.quaternion_rotation_matrix(q / np.linalg.norm(q)))
    assert np.allclose(r @ r.T, np.eye(3), atol=1e-14) and abs(np.linalg.det(r) - 1) < 1e-14


def test_kubric_cameras_flip_and_scale(tmp_path):
    from oracle import pcl_oracle as P
    scene = P.write_kubric_scene(str(tmp_path), "scn00003", 6, 10, 2, 5)
    import json
    meta = json.load(open(os.path.join(scene, "scn00003_p0_v5.json")))
    cams, hw = C.kubric_cameras(scene, 2)
    assert cams.shape == (2, 16, 16) and cams.dtype == np.float32 and hw == (6, 10)
    K = np.abs(np.asarray(meta["camera"]["K"])).astype(np.float32)
    row = cams[1, 5]
    assert row[0] == K[0, 0] * np.float32(10) and row[2] == K[0, 2] * np.float32(10)
    assert row[1] == K[1, 1] * np.float32(6) and row[3] == K[1, 2] * np.float32(6)
    R = C.quaternion_rotation_matrix(meta["camera"]["quaternions"][1]).astype(np.float32)
    R[:, 1:] *= -1
    assert np.array_equal(row[4:13].reshape(3, 3), R)
    assert np.array_equal(row[13:], np.asarray(meta["camera"]["positions"][1], np.float64).astype(np.float32))
    with pytest.raises(ValueError, match="2 frames, the conversion needs 60"):
        C.kubric_cameras(scene)


def test_pardom_view_order(tmp_path):
    from oracle import pcl_oracle as P
    scene = P.write_pardom_scene(str(tmp_path), "scene_000003", 4, 6, 1, 6)
    views = C.pardom_views(scene)
    assert len(views) == 19 and views[16] == "yaw-0" and views[:3] == ["camera0", "camera1", "camera10"]
    cams = C.pardom_cameras(scene, views)
    assert cams.shape == (19, 16)
    with pytest.raises(ValueError, match="no camera for views"):
        C.pardom_cameras(scene, views[:18] + ["camera99"])


def test_discovery_and_skip_rule(tmp_path):
    for d in ("scn00002", "scn00001", "scn00003", "other", "scene_000001"):
        os.makedirs(tmp_path / d)
    assert C.discover_scenes("kubric", str(tmp_path)) == ["scn00001", "scn00002", "scn00003"]
    assert C.discover_scenes("kubric", str(tmp_path), start_idx=1, end_idx=2) == ["scn00002"]
    assert C.discover_scenes("pardom", str(tmp_path)) == ["scene_000001"]
    lst = tmp_path / "list.txt"
    lst.write_text("\n/datasets/Kubric-4D/data/scn02900\n# comment\n/elsewhere/scn02901/\n")
    assert C.discover_scenes("kubric", str(tmp_path), str(lst)) == ["scn02900", "scn02901"]
    out = tmp_path / "out"
    os.makedirs(out)
    for t in range(49):
        (out / f"pcl_rgb_segm_{t * 10 + 5:06d}.pt").write_bytes(b"")
    (out / "pcl_rgb_segm_000495.pt.tmp").write_bytes(b"")
    assert not C.is_finished(str(out), "pardom")
    (out / "pcl_rgb_segm_000495.pt").write_bytes(b"")
    assert C.is_finished(str(out), "pardom") and not C.is_finished(str(out), "kubric")


def test_atomic_save(tmp_path, monkeypatch):
    path = str(tmp_path / "pcl_rgb_segm_00000.pt")
    C.save_frame(path, [torch.ones(2, 3, dtype=torch.float16)])
    assert os.listdir(tmp_path) == ["pcl_rgb_segm_00000.pt"]
    assert torch.equal(torch.load(path, weights_only=True)[0], torch.ones(2, 3, dtype=torch.float16))

    def boom(obj, f):
        f.write(b"partial")
        raise OSError("disk full")
    monkeypatch.setattr(torch, "save", boom)
    with pytest.raises(OSError):
        C.save_frame(str(tmp_path / "pcl_rgb_segm_00001.pt"), [])
    assert sorted(os.listdir(tmp_path)) == ["pcl_rgb_segm_00000.pt", "pcl_rgb_segm_00001.pt.tmp"]
    assert not C.is_finished(str(tmp_path), "kubric")


def test_missing_pardom_frame_is_none(tmp_path):
    from oracle import pcl_oracle as P
    scene = P.write_pardom_scene(str(tmp_path), "scene_000004", 4, 6, 2, 7, missing=(1, "yaw-60"))
    views = C.pardom_views(scene)
    assert C.decode_frame("pardom", C.pardom_frame_paths(scene, views, 1)) is None
    d, rgb, segm = C.decode_frame("pardom", C.pardom_frame_paths(scene, views, 0))
    assert d.shape == (19, 4, 6) and rgb.shape == (19, 24, 3) and segm.shape == (19, 24, 1)


def test_command_line_refusals(tmp_path):
    with pytest.raises(SystemExit):
        C.main(["--kind", "nuscenes", "--input-root", str(tmp_path), "--output-root", str(tmp_path)])
    lst = tmp_path / "l.txt"
    lst.write_text("scn00001\n")
    with pytest.raises(SystemExit, match="exclude each other"):
        C.main(["--kind", "kubric", "--input-root", str(tmp_path), "--output-root", str(tmp_path), "--examples", str(lst),
                "--start-idx", "3"])
    with pytest.raises(SystemExit, match="is not a directory"):
        C.main(["--kind", "kubric", "--input-root", str(tmp_path / "nope"), "--output-root", str(tmp_path)])
    with pytest.raises(SystemExit, match="is not a file"):
        C.main(["--kind", "kubric", "--input-root", str(tmp_path), "--output-root", str(tmp_path), "--examples", str(tmp_path / "x")])
    with pytest.raises(ValueError, match="kind must be"):
        C.convert_scene("nuscenes", str(tmp_path), str(tmp_path))
