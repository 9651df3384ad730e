"""The unprojection kernel (ops.unproject_depth, csrc/unproject.cu) and `python -m gcd_b200.convert` on the device.

Criteria, per element of the stored fp16 xyz:
  * against the float64 oracle (oracle/pcl_oracle.unproject_f64, same float32 inputs):
        |y - ref| <= ulp_fp16(max(|y|, |ref|)) / 2 + KAPPA 2^-24 (sum_j |R_ij c_j| + |t_i|),  KAPPA = 32,
    the fp16 store's half ulp plus the fp32 roundings of the chain (about a dozen in the depth correction and the camera-space point,
    three in the rotation), with NaN positions and +-inf identical;
  * against the reference's float32 torch chain run on this GPU (oracle/pcl_oracle.torch_chain) and against the stored goldens
    (the reference's own CPU run): different on at most ULP_FRAC of the elements, and there at most one fp16 ulp apart unless the
    output cancels: the chains sum `xyz @ R.T` in their BLAS's order (and may contract torch.linspace's product and sum), so two
    fp32 results differ by up to 2 KAPPA 2^-24 (sum_j |R_ij c_j| + |t_i|), which is several fp16 ulps of an output much smaller
    than its terms. Such elements must lie within ulp_fp16 + that. The measured fraction and the count beyond one ulp are printed.
Sizes: the goldens' (16 / 19 views of 12 x 16) and full size (Kubric 16 x 384 x 576, ParDom 19 x 480 x 640).

End to end: the command converts synthetic Kubric and ParDom scenes; evaluate's loaders read the files, the renders of the converted
clouds equal those of the oracle's within max-abs 1e-5 on RENDER_FRAC of the values, a second run skips the finished scene, and the
converted Kubric scene goes through `python -m gcd_b200.evaluate`. tests/test_render_gpu.py asks 99.9 % for renders of identical
clouds; here the two clouds also differ by an ulp on about 0.05 % of the coordinates, and each such point's splat is spread by the
21-tap leak blur over the per-pixel random colours of the synthetic scenes (measured on one H100: 99.86 % for ParDom, 99.90 % for
Kubric at 56 x 84)."""
import json
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu
KAPPA = 32
ULP_FRAC = 1e-3
RENDER_TOL, RENDER_FRAC = 1e-5, 0.997


def kernel(kind, depth, cams):
    from gcd_b200 import convert as C, ops
    d = torch.as_tensor(depth).cuda().contiguous()
    c = torch.as_tensor(cams).cuda().contiguous()
    out = torch.empty((d.shape[0], d.shape[1] * d.shape[2], 3), dtype=torch.float16, device="cuda")
    ops.unproject_depth(d, c, ops.UNPROJECT_BALL_TO_PLANE if kind == "kubric" else ops.UNPROJECT_CLAMP, out,
                        0.0 if kind == "kubric" else C.PARDOM_MAX_DEPTH)
    torch.cuda.synchronize()
    return out.cpu()


def _ordered(h):
    b = h.view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


def within_one_ulp(got, want, scale, what):
    """scale: float64 [V, N, 3] sum_j |R_ij c_j| + |t_i| of each output (pcl_oracle.unproject_f64)."""
    got, want = got.cpu(), want.cpu()
    assert got.shape == want.shape and got.dtype == want.dtype == torch.float16
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    ok = ~torch.isnan(want)
    d = (_ordered(got[ok]) - _ordered(want[ok])).abs()
    frac = (d > 0).double().mean().item()
    far = d > 1
    print(f"{what}: {int((d > 0).sum())} of {d.numel()} elements apart (fraction {frac:.2e}), {int(far.sum())} by more than one "
          f"ulp (max {int(d.max())})")
    assert frac <= ULP_FRAC, what
    if far.any():
        a, b, sc = got[ok][far].double(), want[ok][far].double(), scale[ok][far]
        assert torch.isfinite(a).all() and torch.isfinite(b).all(), what
        bound = ulp_fp16(torch.maximum(a.abs(), b.abs())) + 2 * KAPPA * 2.0 ** -24 * sc
        assert ((a - b).abs() <= bound).all(), what
    return frac


def scales(depth, cams, kind):
    from oracle import pcl_oracle as P
    return torch.stack([P.unproject_f64(depth[j], cams[j], kind)[1] for j in range(depth.shape[0])])


def ulp_fp16(a):
    _, e = torch.frexp(a)
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), torch.ldexp(torch.ones_like(a), e - 11))


def within_f64_bound(got, depth, cams, kind, what):
    from oracle import pcl_oracle as P
    worst = 0.0
    for j in range(got.shape[0]):
        ref, scale = P.unproject_f64(depth[j], cams[j], kind)
        y = got[j].double()
        assert torch.equal(torch.isnan(y), torch.isnan(ref)), (what, j)
        ref16 = ref.to(torch.float16).double()
        for s in (1, -1):
            assert torch.equal(y == s * math.inf, ref16 == s * math.inf), (what, j, s)
        fin = torch.isfinite(y) & torch.isfinite(ref16)
        a, r, sc = y[fin], ref[fin], scale[fin]
        bound = ulp_fp16(torch.maximum(a.abs(), r.abs())) / 2 + KAPPA * 2.0 ** -24 * sc
        ratio = ((a - r).abs() / bound).max().item()
        worst = max(worst, ratio)
    print(f"{what}: worst |y - ref| / bound {worst:.3f} (KAPPA {KAPPA})")
    assert worst <= 1.0, what


def scene_inputs(kind, scene, frames):
    from gcd_b200 import convert as C
    if kind == "kubric":
        cams, _ = C.kubric_cameras(scene, max(frames) + 1)
        return {t: (C.decode_frame(kind, C.kubric_frame_paths(scene, t))[0], cams[t]) for t in frames}
    views = C.pardom_views(scene)
    cams = C.pardom_cameras(scene, views)
    out = {}
    for t in frames:
        got = C.decode_frame(kind, C.pardom_frame_paths(scene, views, t))
        if got is not None:
            out[t] = (got[0], cams)
    return out


@pytest.mark.parametrize("kind", ["kubric", "pardom"])
def test_kernel_golden_size(kind, tmp_path):
    from oracle import pcl_oracle as P, pin_convert as PC
    g = torch.load(os.path.join(GOLD, f"pcl_{kind}.pt"), weights_only=True)
    scene = PC.write_case(str(tmp_path), g["case"])
    for t, (depth, cams) in scene_inputs(kind, scene, sorted(g["frames"])).items():
        got = kernel(kind, depth, cams)
        within_f64_bound(got, depth, cams, kind, f"{kind} golden frame {t} vs float64")
        sc = scales(depth, cams, kind)
        within_one_ulp(got, P.torch_chain(depth, cams, kind, "cuda"), sc, f"{kind} golden frame {t} vs torch chain on the GPU")
        within_one_ulp(got, g["frames"][t][0], sc, f"{kind} golden frame {t} vs the reference's stored xyz")


@pytest.mark.parametrize("kind,hw", [("kubric", (384, 576)), ("pardom", (480, 640))])
def test_kernel_full_size(kind, hw, tmp_path):
    from oracle import pcl_oracle as P
    H, W = hw
    if kind == "kubric":
        scene = P.write_kubric_scene(str(tmp_path), "scn00011", H, W, 1, 41)
    else:
        scene = P.write_pardom_scene(str(tmp_path), "scene_000011", H, W, 1, 42)
    (depth, cams), = scene_inputs(kind, scene, [0]).values()
    assert depth.shape == ((16 if kind == "kubric" else 19), H, W)
    got = kernel(kind, depth, cams)
    within_f64_bound(got, depth, cams, kind, f"full-size {kind} vs float64")
    sc = scales(depth, cams, kind)
    within_one_ulp(got, P.torch_chain(depth, cams, kind, "cuda"), sc, f"full-size {kind} vs torch chain on the GPU")
    within_one_ulp(got, P.torch_chain(depth, cams, kind, "cpu"), sc, f"full-size {kind} vs torch chain on the CPU")


def _render_close(a, b, what):
    d = (a.float().cpu() - b.float().cpu()).abs()
    frac = (d <= RENDER_TOL).double().mean().item()
    print(f"{what}: max-abs {d.max().item():.2e}, fraction within {RENDER_TOL:g}: {frac:.6f}")
    assert frac >= RENDER_FRAC, what


def test_command_line_end_to_end(tmp_path, capsys):
    from gcd_b200 import convert as C, evaluate as E, render
    from oracle import pcl_oracle as P, pin_convert as PC, render_oracle as RO
    import test_evaluate_gpu as TE
    data, pcl = tmp_path / "data", tmp_path / "pcl"
    kub = P.write_kubric_scene(str(data), "scn00001", 24, 36, C.KUBRIC_FRAMES, 51)
    par = P.write_pardom_scene(str(data), "scene_000001", 24, 32, C.PARDOM_FRAMES, 52, missing=(1, "yaw-60"))
    assert C.main(["--kind", "kubric", "--input-root", str(data), "--output-root", str(pcl)]) == 0
    assert C.main(["--kind", "pardom", "--input-root", str(data), "--output-root", str(pcl)]) == 0
    recs = [json.loads(x) for x in capsys.readouterr().out.splitlines() if x.startswith("{")]
    assert [(r["scene"], r["status"]) for r in recs] == [("scn00001", "done"), ("scene_000001", "done")]
    assert recs[0]["frames"] == 60 and recs[1]["frames"] == 49 and recs[1]["skipped_frames"] == [1]
    assert len(os.listdir(pcl / "scn00001")) == 60 and len(os.listdir(pcl / "scene_000001")) == 49

    frames = list(range(2, 2 + 14))
    xyz, rgb = E.load_kubric_clouds(str(pcl / "scn00001"), frames)
    ora = PC.oracle_frames("kubric", kub, frames)
    inp = scene_inputs("kubric", kub, frames)
    for i, t in enumerate(frames):
        within_one_ulp(xyz[i], ora[t][0], scales(*inp[t], "kubric"), f"converted kubric frame {t} vs oracle")
        assert torch.equal(rgb[i], ora[t][1])
    oxyz, orgb = torch.stack([ora[t][0] for t in frames]), torch.stack([ora[t][1] for t in frames])
    K = E.read_kubric_intrinsics(kub)
    src, dst = RO.trajectory(14, 20, 20, 14, 3), RO.trajectory(14, 75, 95, 13, 4)
    hw = dict(render_hw=(56, 84), frame_hw=(48, 72))
    got = render.kubric_views(xyz.cuda(), rgb.cuda(), K, src, dst, True, **hw)
    want = render.kubric_views(oxyz.cuda(), orgb.cuda(), K, src, dst, True, **hw)
    for a, b, w in zip(got, want, ("src", "dst", "reproject")):
        _render_close(a, b, f"converted kubric render {w}")

    xyz, rgb, segm = E.load_pardom_clouds(str(pcl / "scene_000001"), frames)
    ora = PC.oracle_frames("pardom", par, frames)
    inp = scene_inputs("pardom", par, frames)
    for i, t in enumerate(frames):
        within_one_ulp(xyz[i], ora[t][0], scales(*inp[t], "pardom"), f"converted pardom frame {t} vs oracle")
        assert torch.equal(rgb[i], ora[t][1]) and torch.equal(segm[i], ora[t][2])
    Kp = E.read_pardom_intrinsics(par)[16].clone()
    Kp[0] /= 32.0
    Kp[1] /= 24.0
    intr, ext = Kp[None].repeat(14, 1, 1), RO.trajectory(14, 10, 30, 14, 3)
    got = render.pardom_views(xyz.cuda(), rgb.cuda(), intr, ext, "rgb", segm.cuda(), None, 0, True, **hw)
    want = render.pardom_views(torch.stack([ora[t][0] for t in frames]).cuda(), torch.stack([ora[t][1] for t in frames]).cuda(),
                               intr, ext, "rgb", torch.stack([ora[t][2] for t in frames]).cuda(), None, 0, True, **hw)
    for a, b, w in zip(got, want, ("rgb", "reproject")):
        _render_close(a, b, f"converted pardom render {w}")

    assert C.main(["--kind", "kubric", "--input-root", str(data), "--output-root", str(pcl)]) == 0
    rec = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert rec["scene"] == "scn00001" and rec["status"] == "skipped"

    ck = str(tmp_path / "tiny.ckpt")
    gold = TE._write_checkpoint(ck)
    mc = tmp_path / "model.json"
    mc.write_text(json.dumps({"unet": {"model_channels": 64}, "vae": {"ch": 64}, "encoder": gold["enc_cfg"], "vit": gold["vit_cfg"]}))
    (tmp_path / "list.txt").write_text(kub + "\n")
    ctl = {"scn00001": {"sample_00": {"frame_start": 2, "frame_skip": 1, "spherical_start": [20.0, 10.0, 15.0],
                                      "spherical_end": [50.0, 25.0, 15.0]}}}
    (tmp_path / "controls.json").write_text(json.dumps(ctl))
    out = tmp_path / "out"
    summary = E.main(["--kind", "kubric", "--checkpoint", ck, "--model-config", str(mc), "--examples", str(tmp_path / "list.txt"),
                      "--pcl-root", str(pcl), "--control-json", str(tmp_path / "controls.json"), "--output", str(out),
                      "--num-samples", "2", "--num-steps", "2", "--frame-height", str(TE.FRAME_HW[0]), "--frame-width",
                      str(TE.FRAME_HW[1]), "--render-height", str(TE.RENDER_HW[0]), "--render-width", str(TE.RENDER_HW[1])])
    d = json.loads((out / "000_scn00001_c00_metrics.json").read_text())
    assert all(math.isfinite(v) for v in d["mean_psnr"]) and math.isfinite(summary["mean_psnr"])


def test_failed_scene_exits_nonzero(tmp_path, capsys):
    from gcd_b200 import convert as C
    from oracle import pcl_oracle as P
    data = tmp_path / "data"
    P.write_pardom_scene(str(data), "scene_000002", 4, 6, 1, 61)          # one frame only: frames 1..49 missing, skipped
    os.makedirs(data / "scene_000003" / "rgb")                              # no views: fails
    with pytest.raises(SystemExit) as e:
        C.main(["--kind", "pardom", "--input-root", str(data), "--output-root", str(tmp_path / "pcl")])
    assert e.value.code == 1
    cap = capsys.readouterr()
    recs = [json.loads(x) for x in cap.out.splitlines() if x.startswith("{")]
    assert [(r["scene"], r["status"]) for r in recs] == [("scene_000002", "done"), ("scene_000003", "failed")]
    assert recs[0]["frames"] == 1 and "scene_000003" in cap.err
