"""Point-cloud view synthesis, CPU side: the torch restatement (oracle/render_oracle.py) against the reference's own outputs
(tests/golden/render_*.pt, written by oracle/pin_render.py from the reference's geometry.py / synth_* code run on CPU), the public
API's argument checks, and spreaded_index_add's offsets. The oracle reproduces the reference bit for bit on the goldens' machine;
1e-6 leaves room for another BLAS summing the 3x3 projections in another order."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def test_oracle_matches_reference_goldens():
    from oracle import pin_render as PR
    from oracle import render_oracle as O
    g = torch.load(os.path.join(GOLD, "render_kubric.pt"))
    cl, src, dst = PR.kubric_case(g["case"])
    s, d, r = O.kubric_views(cl["xyz"], cl["rgb"], cl["intrinsics"][0], src, dst, True, g["meta"]["render_hw"],
                             g["meta"]["frame_hw"])
    for a, k in ((s, "rgb_src"), (d, "rgb_dst"), (r, "reproject")):
        err = (a - g[k]).abs().max().item()
        print(f"kubric {k}: max-abs {err:.2e}")
        assert err <= 1e-6
    g = torch.load(os.path.join(GOLD, "render_pardom.pt"))
    cl, ext = PR.pardom_case(g["case"])
    for name, modality, mt, rep in (("rgb", "rgb", 0, True), ("segm0", "segm", 0, False), ("segm2", "segm", 2, True)):
        o, rp = O.pardom_views(cl["xyz"], cl["rgb"], cl["intrinsics"], ext, modality, cl["segm"], cl["palette"], mt, rep,
                               g["meta"]["render_hw"], g["meta"]["frame_hw"])
        assert (o - g[name]).abs().max().item() <= 1e-6
        if rep:
            assert (rp - g[name + "_reproject"]).abs().max().item() <= 1e-6
    assert not torch.isfinite(cl["xyz"].float()).all()          # the ParDom clouds carry fp16-overflowed far points


def test_goldens_small_and_from_reference():
    for f in ("render_kubric.pt", "render_pardom.pt"):
        path = os.path.join(GOLD, f)
        assert os.path.getsize(path) < 1 << 20
        assert "device = 'cpu'" in torch.load(path)["meta"]["edit"]


def test_spread_offsets():
    from oracle.render_oracle import spread_offsets
    assert spread_offsets(0) == []
    assert sorted(spread_offsets(1)) == [(0, 1), (1, 0), (1, 1)]
    assert sorted(spread_offsets(2)) == sorted([(-1, 0), (1, 0), (0, -1), (0, 1), (-1, -1), (-1, 1), (1, -1), (1, 1)])
    o3 = spread_offsets(3)
    assert len(o3) == 15 and {dx for dx, _ in o3} == {-1, 0, 1, 2} and {dy for _, dy in o3} == {-1, 0, 1, 2}


def test_api_rejects_cpu_tensors_and_bad_shapes():
    from gcd_b200 import render
    from gcd_b200._lib import GcdError
    T, V, N = 2, 5, 10
    xyz = torch.zeros(T, V, N, 3, dtype=torch.float16)
    rgb = torch.zeros(T, V, N, 3, dtype=torch.uint8)
    ext = torch.eye(4).expand(T, 4, 4)
    K = torch.eye(3)
    with pytest.raises(GcdError):
        render.kubric_views(xyz, rgb, K, ext, ext, render_hw=(28, 42), frame_hw=(24, 36))
    with pytest.raises(GcdError):
        render.render_views(xyz[:, 0], rgb[:, 0], K, ext, (28, 42), (24, 36), 1, 21)
    with pytest.raises(GcdError):
        render.pardom_views(xyz, rgb, K.expand(T, 3, 3), ext)
    with pytest.raises(ValueError):
        render.kubric_views(xyz[0], rgb[0], K, ext, ext)                       # no frame axis
    with pytest.raises(ValueError):
        render.kubric_views(xyz, rgb[:, :, :-1], K, ext, ext)                   # rgb / xyz mismatch
    with pytest.raises(ValueError):
        render.kubric_views(xyz, rgb, K, ext[:1], ext)                          # one camera short
    with pytest.raises(ValueError):
        render.kubric_views(xyz[:, :4], rgb[:, :4], K, ext, ext, reproject=True)  # view 4 missing
    with pytest.raises(ValueError):
        render.pardom_views(xyz, rgb, K.expand(T, 3, 3), ext, modality="depth")
    with pytest.raises(ValueError):
        render.pardom_views(xyz, rgb, K.expand(T, 3, 3), ext, modality="segm")  # no segm / palette
    with pytest.raises(ValueError):
        render.render_views(xyz[:, 0], rgb[:, 0], K, ext[:1].expand(3, 4, 4), (28, 42), (24, 36), 1, 21)
