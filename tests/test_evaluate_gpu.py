"""gcd_b200.evaluate on the device: S samples as S clips of one sampler run against S sequential sample_video calls on the same
noise, the metrics dict of one example, and the command line end to end on written synthetic examples. Tiny seeded UNet, decoder,
encoder and CLIP tower (as in tests/test_clip_gpu.py), a synthetic point cloud (oracle/render_oracle.synthetic_clouds).

Tolerance. The batched run need not be bit-identical to the sequential one: the fused GroupNorm statistics of a 3-clip batch may
be summed in another order than those of a 1-clip batch (DESIGN.md §3, §7). Latents and frames agree within relative L2 TOL (the
measured values are printed; 0 at this size on one H100, 3.4e-4 at 256 x 384 with the full-width UNet); a wrong noise /
conditioning pairing gives errors of order one."""
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
TOL = 1e-2
T, S, STEPS = 14, 3, 4
FRAME_HW, RENDER_HW = (64, 128), (70, 140)     # latent 8 x 16: three UNet levels halve it
ANGLES = (20.0, 30.0, 10.0, 15.0, 15.0, 0.0)


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _cond_gold():
    return torch.load(os.path.join(GOLD, "cond_kubric_tiny.pt"))


def _hot_path():
    from gcd_b200 import spec, synthetic
    from gcd_b200.clip import visual_param_shapes
    from gcd_b200.pipeline import GCDHotPath
    gold = _cond_gold()
    pipe = GCDHotPath(spec.UNET_TINY, spec.VAE_TINY, num_steps=STEPS, num_frames=T, device="cuda")
    vst = synthetic.seeded_state(visual_param_shapes(gold["vit_cfg"]), seed=gold["vit_seed"])
    pipe.load_clip({"model.visual." + k: v for k, v in vst.items()}, vit_cfg=gold["vit_cfg"])
    pipe.load_cond_encoder(synthetic.seeded_state(spec.encoder_param_shapes(gold["enc_cfg"]), seed=gold["enc_seed"]),
                           gold["quant_w"], gold["quant_b"], enc_cfg=gold["enc_cfg"])
    pipe.load_spherical(gold["sph_w"], gold["sph_b"])
    pipe.load_state(synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_TINY), seed=0),
                    synthetic.seeded_state(spec.decoder_param_shapes(spec.VAE_TINY), seed=0))
    return pipe


def _lpips():
    from gcd_b200.lpips import LPIPS
    from oracle import lpips_oracle as O
    m = LPIPS()
    m.load_state_dict(O.seeded_state(0))
    return m.cuda()


def _example(seed=21):
    from gcd_b200 import evaluate as E, render
    from oracle import render_oracle as RO
    cl = RO.synthetic_clouds("kubric", T, 16, 24, 36, seed)
    row = E.control_row("kubric", None, 0, 2, 12, ANGLES)
    traj = E.kubric_trajectories(row)
    src, dst, rep = render.kubric_views(cl["xyz"].cuda(), cl["rgb"].cuda(), cl["intrinsics"][0], traj["extrinsics_src"],
                                        traj["extrinsics_dst"], True, RENDER_HW, FRAME_HW)
    batch = E.construct_batch("kubric", traj, src, dst, rep, 12, torch.Generator(device="cuda").manual_seed(seed))
    return (batch["jpg"], batch["reproject"]), batch


@pytest.fixture(scope="module")
def run():
    from gcd_b200 import evaluate as E
    pipe, lp = _hot_path(), _lpips()
    views, batch = _example()
    samples, m, unc = E.evaluate_example(pipe, views, batch, S, torch.Generator(device="cuda").manual_seed(5), lpips=lp)
    g = torch.Generator(device="cuda").manual_seed(5)
    seq = []
    for _ in range(S):                                  # test.py's run_inference: condition + sample_video per sample
        c, uc = pipe.condition(batch)
        noise = torch.randn((T, 4, FRAME_HW[0] // 8, FRAME_HW[1] // 8), generator=g, device="cuda")
        z, x = pipe.sample_video(noise, c, uc)
        seq.append((z, torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0)))
    return dict(pipe=pipe, lp=lp, views=views, batch=batch, samples=samples, m=m, unc=unc, seq=seq)


def test_batched_samples_match_sequential_sample_video(run):
    assert run["pipe"].sampler.last_path == "fused"
    assert len(run["samples"]) == S
    for s, (d, (z, x)) in enumerate(zip(run["samples"], run["seq"])):
        assert d["sampled_latent"].shape == (T, 4, FRAME_HW[0] // 8, FRAME_HW[1] // 8) and d["sampled_rgb"].shape == (T, 3, *FRAME_HW)
        assert d["cond_rgb"].shape == (T, 3, *FRAME_HW) and 0 <= d["cond_rgb"].min() and d["cond_rgb"].max() <= 1
        ez, ex = relerr(d["sampled_latent"], z), relerr(d["sampled_rgb"], x)
        print(f"sample {s}: latents rel-L2 {ez:.2e}, frames rel-L2 {ex:.2e} (batched vs sequential)")
        assert ez < TOL and ex < TOL
    # the samples differ from each other: each got its own noise
    assert relerr(run["samples"][0]["sampled_latent"], run["samples"][1]["sampled_latent"]) > 0.1


def test_metrics_dict_matches_calculate_metrics_of_sequential_outputs(run):
    from gcd_b200 import evaluate as E, metrics
    m = run["m"]
    assert set(m) == set(E.METRIC_KEYS + E.MASKED_METRIC_KEYS + E.LPIPS_KEYS)
    for k, v in m.items():
        want = {"frame_diversity": (T,), "mean_diversity": ()}.get(k.replace("_vis", "").replace("_occ", ""))
        if want is None:
            want = (S, T) if k.startswith("frame_") else (S,)
        assert tuple(v.shape) == want, (k, tuple(v.shape))
    rep01 = (run["views"][1] + 1) / 2
    occ = (rep01.abs().sum(dim=1) <= 1e-7).cpu()
    vis_empty, occ_empty = (~occ).flatten(1).sum(1) == 0, occ.flatten(1).sum(1) == 0
    print(f"occluded pixels per frame: {occ.flatten(1).sum(1).tolist()}")
    for k, v in m.items():
        if k.endswith("_occ") and k.startswith("frame_") and "diversity" not in k:
            assert torch.equal(torch.isnan(v), occ_empty[None].expand(S, T)), k
        elif k.endswith("_vis") and k.startswith("frame_") and "diversity" not in k:
            assert torch.equal(torch.isnan(v), vis_empty[None].expand(S, T)), k
        elif k.startswith("frame_") and "diversity" not in k:
            assert torch.isfinite(v).all(), k
    gt01 = (run["views"][0] + 1) / 2
    ref, _ = metrics.calculate_metrics(gt01, rep01, torch.stack([x for _, x in run["seq"]]), lpips=run["lp"])
    for k in ("frame_psnr", "frame_ssim", "frame_lpips", "frame_psnr_vis", "frame_ssim_occ"):
        a, b = m[k], ref[k]
        ok = torch.isnan(a) == torch.isnan(b)
        assert ok.all(), k
        d = (a - b).abs()[~torch.isnan(b)].max().item()
        bound = 0.05 if "psnr" in k else 1e-2
        print(f"{k}: max |batched - sequential| {d:.2e} (bound {bound})")
        assert d < bound, k


def _write_example(root, pcl_root, name, seed):
    from oracle import render_oracle as RO
    cl = RO.synthetic_clouds("kubric", T, 16, 24, 36, seed)
    scene = os.path.join(root, name)
    os.makedirs(scene)
    with open(os.path.join(scene, f"{name}_p0_v4.json"), "w") as f:
        json.dump({"camera": {"K": cl["intrinsics"][0].tolist()}}, f)
    pdir = os.path.join(pcl_root, name)
    os.makedirs(pdir)
    for t in range(T):
        torch.save([cl["xyz"][t], cl["rgb"][t], torch.zeros_like(cl["rgb"][t])], os.path.join(pdir, f"pcl_rgb_segm_{2 + t:05d}.pt"))
    return scene


def _write_checkpoint(path):
    from gcd_b200 import checkpoint, embedders, spec, synthetic
    from gcd_b200.lpips import LPIPS
    from gcd_b200.unet import VideoUNet
    from gcd_b200.vae import VideoDecoder
    from oracle import lpips_oracle as O
    gold = _cond_gold()
    embs = embedders.build_embedders(embedders.gcd_conditioner_config(spherical=True, vit_cfg=gold["vit_cfg"],
                                                                      enc_cfg=gold["enc_cfg"]))
    root = checkpoint.HotPathRoot(VideoUNet(**spec.unet_ctor_kwargs(spec.UNET_TINY)),
                                  VideoDecoder(**spec.decoder_ctor_kwargs(spec.VAE_TINY)), conditioner=embs, lpips=LPIPS())
    lp = {"lpips." + k: v for k, v in O.seeded_state(0).items()}
    sd = {k: (lp[k] if k in lp else synthetic.seeded_tensor(k, v.shape, seed=0)) for k, v in root.state_dict().items()}
    torch.save({"state_dict": sd}, path)
    return gold


def test_command_line_end_to_end(tmp_path):
    from gcd_b200 import evaluate as E
    ck = str(tmp_path / "tiny.ckpt")
    gold = _write_checkpoint(ck)
    mc = tmp_path / "model.json"
    mc.write_text(json.dumps({"unet": {"model_channels": 64}, "vae": {"ch": 64}, "encoder": gold["enc_cfg"], "vit": gold["vit_cfg"]}))
    names = ["scn00001", "scn00002"]
    scenes = [_write_example(str(tmp_path / "data"), str(tmp_path / "pcl"), n, 30 + i) for i, n in enumerate(names)]
    (tmp_path / "list.txt").write_text("\n".join(scenes) + "\n")
    ctl = {n: {"sample_00": {"frame_start": 2, "frame_skip": 1, "spherical_start": [20.0, 10.0, 15.0],
                             "spherical_end": [50.0 + 10 * i, 25.0, 15.0]}} for i, n in enumerate(names)}
    (tmp_path / "controls.json").write_text(json.dumps(ctl))
    out = tmp_path / "out"
    summary = E.main(["--kind", "kubric", "--checkpoint", ck, "--model-config", str(mc), "--examples", str(tmp_path / "list.txt"),
                      "--pcl-root", str(tmp_path / "pcl"), "--control-json", str(tmp_path / "controls.json"), "--output", str(out),
                      "--num-samples", "2", "--num-steps", "2", "--frame-height", str(FRAME_HW[0]), "--frame-width",
                      str(FRAME_HW[1]), "--render-height", str(RENDER_HW[0]), "--render-width", str(RENDER_HW[1])])
    files = sorted(p.name for p in out.iterdir())
    assert files == ["000_scn00001_c00_metrics.json", "001_scn00002_c00_metrics.json", "summary_rank0.json"], files
    for f in files[:2]:
        d = json.loads((out / f).read_text())
        assert list(d) == list(E.METRIC_KEYS + E.MASKED_METRIC_KEYS + E.LPIPS_KEYS)
        assert len(d["frame_psnr"]) == 2 and len(d["frame_psnr"][0]) == T and all(math.isfinite(v) for v in d["mean_psnr"])
    s = json.loads((out / "summary_rank0.json").read_text())
    assert s["examples"] == 2 and math.isfinite(s["mean_psnr"]) and s["mean_psnr"] == summary["mean_psnr"]
