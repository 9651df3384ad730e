"""Point-cloud view synthesis on the device (gcd_b200.render, csrc/render.cu) against the reference's outputs (tests/golden/render_*.pt)
and the live torch oracle (oracle/render_oracle.py).

Tolerances. The kernels keep the reference's fp64 accumulation, but the results are not bit-exact:
  * fp64 atomics add the splats in a scheduling-dependent order (relative 1e-16 on the weight sums);
  * the leak blur runs separably in fp64 where the reference convolves the float32 image with a float32 2-D kernel (relative ~1e-7);
  * a point whose fp64 `uv + 0.5` lies within an ulp of an integer can truncate to the neighbouring pixel when the 3x3 products are
    summed in another order than torch.mm's; that moves one splat and the pixels its blur reaches.
So: max-abs <= 1e-5 on at least 99.9 % of the output values, the occluded mask (reprojection == 0, test.py:366) identical on at least
99.99 % of the pixels. The measured values are printed."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu
TOL, FRAC, MASK_FRAC = 1e-5, 0.999, 0.9999


def close(got, want, what):
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = (got - want).abs()
    frac = (d <= TOL).double().mean().item()
    print(f"{what}: max-abs {d.max().item():.2e}, fraction within {TOL:g}: {frac:.6f}")
    assert frac >= FRAC, (what, frac)


def occluded(rep):
    return ((rep.float().cpu() + 1) / 2).abs().sum(dim=1) <= 1e-7


def same_mask(got, want, what):
    a, b = occluded(got), occluded(want)
    frac = (a == b).double().mean().item()
    print(f"{what} occluded mask: agreement {frac:.6f} ({int(b.sum())} occluded pixels)")
    assert frac >= MASK_FRAC


def cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def test_kubric_views_vs_reference_golden():
    from gcd_b200 import render
    from oracle import pin_render as PR
    g = torch.load(os.path.join(GOLD, "render_kubric.pt"))
    cl, src, dst = PR.kubric_case(g["case"])
    c = cuda(cl)
    s, d, r = render.kubric_views(c["xyz"], c["rgb"], cl["intrinsics"][0], src, dst, True, g["meta"]["render_hw"],
                                  g["meta"]["frame_hw"])
    close(s, g["rgb_src"], "kubric rgb_src")
    close(d, g["rgb_dst"], "kubric rgb_dst")
    close(r, g["reproject"], "kubric reproject")
    same_mask(r, g["reproject"], "kubric")
    s2, d2, r2 = render.kubric_views(c["xyz"], c["rgb"], cl["intrinsics"][0], src, dst, False, g["meta"]["render_hw"],
                                     g["meta"]["frame_hw"])
    assert r2 is None
    close(s2, g["rgb_src"], "kubric rgb_src without reprojection")


def test_pardom_views_vs_reference_golden():
    from gcd_b200 import render
    from oracle import pin_render as PR
    g = torch.load(os.path.join(GOLD, "render_pardom.pt"))
    cl, ext = PR.pardom_case(g["case"])
    c = cuda(cl)
    for name, modality, mt, rep in (("rgb", "rgb", 0, True), ("segm0", "segm", 0, False), ("segm2", "segm", 2, True)):
        o, rp = render.pardom_views(c["xyz"], c["rgb"], cl["intrinsics"], ext, modality, c["segm"], c["palette"], mt, rep,
                                    g["meta"]["render_hw"], g["meta"]["frame_hw"])
        close(o, g[name], f"pardom {name}")
        if rep:
            close(rp, g[name + "_reproject"], f"pardom {name} reproject")
            same_mask(rp, g[name + "_reproject"], f"pardom {name}")
        else:
            assert rp is None


def test_full_size_frames_vs_oracle():
    """One Kubric frame (16 views of 384 x 576 points) and one ParDom frame (19 views of 480 x 640) at 280 x 420 -> 256 x 384."""
    from gcd_b200 import render
    from oracle import render_oracle as O
    cl = O.synthetic_clouds("kubric", 1, 16, 384, 576, seed=21)
    src, dst = O.trajectory(1, 20, 20, 14, 3), O.trajectory(1, 75, 75, 13, 4)
    want = O.kubric_views(cl["xyz"], cl["rgb"], cl["intrinsics"][0], src, dst, True)
    got = render.kubric_views(cl["xyz"].cuda(), cl["rgb"].cuda(), cl["intrinsics"][0], src, dst, True)
    for a, b, w in zip(got, want, ("src", "dst", "reproject")):
        close(a, b, f"full-size kubric {w}")
    same_mask(got[2], want[2], "full-size kubric")
    cl = O.synthetic_clouds("pardom", 1, 19, 480, 640, seed=22)
    ext = O.trajectory(1, 16 / 19 * 360, 16 / 19 * 360, 14, 3)
    want = O.pardom_views(cl["xyz"], cl["rgb"], cl["intrinsics"], ext, "segm", cl["segm"], cl["palette"], 0, True)
    got = render.pardom_views(cl["xyz"].cuda(), cl["rgb"].cuda(), cl["intrinsics"], ext, "segm", cl["segm"].cuda(),
                              cl["palette"].cuda(), 0, True)
    close(got[0], want[0], "full-size pardom segm")
    close(got[1], want[1], "full-size pardom reproject")
    same_mask(got[1], want[1], "full-size pardom")


def test_batched_frames_match_per_frame_calls():
    from gcd_b200 import render
    from oracle import render_oracle as O
    T = 14
    cl = O.synthetic_clouds("kubric", T, 16, 24, 36, seed=31)
    K = O.pixel_intrinsics(cl["intrinsics"][0], (56, 84), 1.5).cuda()
    ext = O.trajectory(T, 0, 90, 14, 3).cuda()
    xyz, rgb = cl["xyz"].reshape(T, -1, 3).cuda(), cl["rgb"].reshape(T, -1, 3).cuda()
    batched = render.render_views(xyz, rgb, K, ext, (56, 84), (48, 72), 1, 21)
    single = torch.cat([render.render_views(xyz[t:t + 1], rgb[t:t + 1], K, ext[t], (56, 84), (48, 72), 1, 21) for t in range(T)])
    d = (batched - single).abs().max().item()
    print(f"batched vs per-frame: max-abs {d:.2e}")
    assert d <= 1e-6


def _edge(scale):
    from oracle import pin_render as PR
    xyz, rgb, K, RT, hw = PR.edge_cloud()
    return (xyz.float() * scale).to(torch.float16), rgb, K, RT, hw


@pytest.mark.parametrize("scale", [1.0, 8.0])       # max depth 12 (Kubric branch, strength 512) and 96 (ParDom branch, 256)
def test_edge_cases_vs_oracle(scale):
    """Points behind / too near the camera, uv in (-1.5, -0.5) (truncation puts them in column / row 0), non-finite fp16 coordinates;
    render size equal to the frame size (the resize is the identity) and a ragged one; spread radius 1, 2 and 3."""
    from gcd_b200 import render
    from oracle import render_oracle as O
    xyz, rgb, K, RT, (H, W) = _edge(scale)
    col = (rgb / 255.0).to(torch.float32)
    assert O.project(xyz.float(), col, K, RT, H, W, 1)[:, 0].sum() > 0     # column 0 is populated
    for frame_hw, rad in (((H, W), 1), ((17, 29), 2), ((H, W), 3)):
        want = O.render(xyz.float(), col, K, RT, (H, W), frame_hw, rad, 21) * 2 - 1
        got = render.render_views(xyz[None].cuda(), rgb[None].cuda(), K, RT, (H, W), frame_hw, rad, 21)[0]
        close(got, want, f"edge x{scale} -> {frame_hw} radius {rad}")


def test_no_point_in_image_raises():
    from gcd_b200 import render
    xyz, rgb, K, RT, (H, W) = _edge(1.0)
    behind = xyz.clone()
    behind[:, 2] = -behind[:, 2].abs()
    both = torch.stack([xyz, behind]).cuda()
    with pytest.raises(ValueError, match="no point"):
        render.render_views(both, torch.stack([rgb, rgb]).cuda(), K, RT, (H, W), (H, W), 1, 21)


def test_eval_loop_masks_and_metrics():
    """Render a clip, feed (rgb_dst + 1) / 2, (reproject + 1) / 2 and S perturbed copies to calculate_metrics, and compare the masks
    and every key with scripts/test.py:346-496's numpy formulas applied to the reference's golden outputs."""
    from gcd_b200 import metrics, render
    from oracle import metrics_oracle as M
    from oracle import pin_render as PR
    g = torch.load(os.path.join(GOLD, "render_kubric.pt"))
    cl, src, dst = PR.kubric_case(g["case"])
    c = cuda(cl)
    _, d, r = render.kubric_views(c["xyz"], c["rgb"], cl["intrinsics"][0], src, dst, True, g["meta"]["render_hw"],
                                  g["meta"]["frame_hw"])
    S = 3
    gen = torch.Generator().manual_seed(4)
    gt_ref, rep_ref = ((g["rgb_dst"] + 1) / 2).numpy(), ((g["reproject"] + 1) / 2).numpy()
    noise = 0.05 * torch.randn(S, *gt_ref.shape, generator=gen)
    pred = (torch.from_numpy(gt_ref)[None] + noise).clamp(0, 1)
    out, unc = metrics.calculate_metrics((d + 1) / 2, (r + 1) / 2, pred.cuda())

    occ = (np.sum(np.abs(rep_ref), axis=1) <= 1e-7).astype(np.uint8)          # test.py:366-368
    vis = 1 - occ
    got_occ = (((r + 1) / 2).abs().sum(dim=1) <= 1e-7).cpu().numpy()
    agree = (got_occ == occ.astype(bool)).mean()
    print(f"eval-loop occluded mask agreement {agree:.6f}, occluded share {occ.mean():.3f}")
    assert agree >= MASK_FRAC and 0 < occ.mean() < 1
    p = pred.numpy()
    T = gt_ref.shape[0]
    want = {k: np.zeros((S, T)) for k in ("frame_psnr", "frame_ssim", "frame_psnr_vis", "frame_ssim_vis", "frame_psnr_occ",
                                          "frame_ssim_occ")}
    for s in range(S):
        for t in range(T):
            want["frame_psnr"][s, t] = M.psnr(p[s, t], gt_ref[t])
            want["frame_ssim"][s, t] = M.ssim_pair(p[s, t], gt_ref[t])[0]
            for name, m in (("vis", vis[t]), ("occ", occ[t])):
                mb = np.tile(m[None].astype(bool), (3, 1, 1))
                want[f"frame_psnr_{name}"][s, t] = M.psnr(p[s, t][mb], gt_ref[t][mb]) if mb.any() else np.nan
                want[f"frame_ssim_{name}"][s, t] = M.ssim_pair(p[s, t], gt_ref[t], m)[1]
    uncertainty = np.nanmean(np.std(p, axis=0), axis=1)
    want["frame_diversity"] = np.nanmean(uncertainty, axis=(1, 2))
    for name, m in (("vis", vis), ("occ", occ)):
        mb = np.tile(m[:, None].astype(bool), (1, 3, 1, 1))
        want[f"frame_diversity_{name}"] = np.array([np.nanmean(np.std(np.stack([x[t][mb[t]] for x in p]), axis=0))
                                                    for t in range(T)])
    for k in list(want):
        want[k.replace("frame_", "mean_")] = np.nanmean(want[k], axis=-1)
    assert set(out) == set(want), set(out) ^ set(want)
    # the rendered target differs from the golden by <= 1e-5 on almost all values; PSNR moves by ~1e-3 dB for that, SSIM by ~1e-5
    tol = {"psnr": 5e-3, "ssim": 5e-5, "diversity": 1e-6}
    for k, v in want.items():
        t = tol[next(x for x in tol if x in k)]
        err = np.nanmax(np.abs(np.asarray(out[k], dtype=np.float64) - v))
        print(f"{k}: max-abs {err:.2e}")
        assert err <= t, (k, err)
    assert tuple(unc.shape) == gt_ref.shape[:1] + gt_ref.shape[2:]
