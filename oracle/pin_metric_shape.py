"""Reference goldens AT THE METRIC SHAPE (TEST INFRASTRUCTURE; needs a reference checkout: GCD_REFERENCE, see oracle/ref_shim.py).

    python -m oracle.pin_metric_shape [unet_kubric] [unet_pardom] [traj25] [traj50] [vae_fullres]     (default: all)

Everything stored is an output of the REFERENCE's own modules (imported through oracle/ref_shim.py) on CPU fp32 with the
seeded weights / inputs of oracle/weights.py — the CUDA path is compared with these in tests/test_metric_shape_gpu.py:

  unet_{kubric,pardom}_metric.pt  one CFG forward (28 frames) of the full-width VideoUNet at latent 72x128, the shape
                                  bench.py measures (video_model.py:461-540): M=258 048-row GEMM tiles, 9216-token
                                  attention, T=14 temporal GroupNorm. Stored as net_out[:, :, ::2, ::4].
  traj25.pt                       the complete 25-step EulerEDMSampler trajectory (sampling.py:123-144) at 14x32x48, full
                                  width, LinearPredictionGuider 1.0 -> 1.5 (BASELINE.md §4.4); x after steps 1, 5, 10, 25 (every 2nd column).
  traj50.pt                       config 4: 50 steps, guider max scale 2.5, at 14x16x24, full width; x after 1, 10, 25, 50.
  vae_fullres.pt                  VideoDecoder (temporal_ae.py:293-349) of 14 frames at latent 72x128 -> 576x1024 px, stored
                                  as a 16x strided subsample + three full-resolution 64x64 crops + per-frame moments.
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gcd_oracle as O  # noqa: E402
from oracle import ref_shim, weights  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_grad_enabled(False)

CROPS = [(0, 0, 0), (7, 256, 480), (13, 512, 960)]          # (frame, y0, x0) of the 64x64 full-resolution crops


def _loaded_ref_unet(cfg):
    net = ref_shim.build_ref_unet(cfg)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    sd = weights.seeded_state(shapes, seed=0)
    net.load_state_dict(sd, strict=True)
    return net


def pin_unet_metric(tag, cfg, T=14, H=72, W=128):
    t0 = time.time()
    net = _loaded_ref_unet(cfg)
    x, c, uc, ioi = weights.seeded_inputs(cfg, 1, T, H, W)
    sigma = torch.full((2 * T,), 10.0)
    c_cat = {k: torch.cat((uc[k], c[k]), 0) for k in c}
    cs, co, ci, cn = O.vscaling_edm_cnoise(sigma.view(-1, 1, 1, 1))
    xin = torch.cat((torch.cat([x, x]) * 3.0 * ci, c_cat["concat"]), 1)
    out = net(xin, cn.reshape(-1), context=c_cat["crossattn"], y=c_cat["vector"], image_only_indicator=ioi,
              num_video_frames=T)
    print(f"[unet {tag} metric] reference forward {tuple(out.shape)} in {time.time() - t0:.0f} s, rms {out.pow(2).mean().sqrt():.4f}",
          flush=True)
    torch.save({"cfg": cfg, "B": 1, "T": T, "H": H, "W": W, "sigma": 10.0, "x_mul": 3.0, "net_out_sub": out[:, :, ::2, ::4].clone()},
               os.path.join(GOLD, f"unet_{tag}_metric.pt"))


def pin_traj(tag, cfg, T, H, W, steps, max_scale, keep, w_stride=1):
    t0 = time.time()
    net = _loaded_ref_unet(cfg)
    from sgm.modules.diffusionmodules.denoiser import Denoiser
    from sgm.modules.diffusionmodules.sampling import EulerEDMSampler
    from sgm.modules.diffusionmodules.wrappers import OpenAIWrapper
    den = Denoiser({"target": "sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise"})
    wrapped = OpenAIWrapper(net)
    x, c, uc, ioi = weights.seeded_inputs(cfg, 1, T, H, W)
    extra = dict(image_only_indicator=ioi, num_video_frames=T)
    sampler = EulerEDMSampler(
        discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.EDMDiscretization",
                               "params": {"sigma_max": 700.0}},
        num_steps=steps,
        guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                       "params": {"num_frames": T, "max_scale": max_scale, "min_scale": 1.0}},
        device="cpu")
    seen = []          # the denoiser's input at call i is cat([x_i] * 2): x_i = state BEFORE step i (x_0 = scaled noise)

    def denoiser_fn(inp, sig, cc):
        seen.append(inp[:T].clone())
        print(f"  [{tag}] step {len(seen)}/{steps}  sigma {sig[0].item():.4f}  ({time.time() - t0:.0f} s)", flush=True)
        return den(wrapped, inp, sig, cc, **extra)

    final = sampler(denoiser_fn, x.clone(), cond=c, uc=uc)
    states = {k: (seen[k] if k < steps else final)[..., ::w_stride].clone() for k in keep}      # x after k steps
    torch.save({"cfg": cfg, "B": 1, "T": T, "H": H, "W": W, "steps": steps, "max_scale": max_scale, "min_scale": 1.0,
                "after_steps": states, "sampled": final[..., ::w_stride].clone(), "w_stride": w_stride},
               os.path.join(GOLD, f"{tag}.pt"))
    print(f"[{tag}] reference {steps}-step trajectory at {T}x{H}x{W} in {time.time() - t0:.0f} s; |x| {final.abs().mean():.4f}", flush=True)


def pin_decoder_fullres(T=14, H=72, W=128):
    t0 = time.time()
    cfg = O.VAE_DECODER
    dec = ref_shim.build_ref_decoder(cfg)
    shapes = {k: tuple(v.shape) for k, v in dec.state_dict().items()}
    dec.load_state_dict(weights.seeded_state(shapes, seed=0), strict=True)
    g = torch.Generator().manual_seed(4321)
    z = torch.randn(T, cfg["z_channels"], H, W, generator=g)
    out = dec(z / 0.18215, timesteps=T)                                   # [14, 3, 576, 1024]
    crops = [out[f, :, y0:y0 + 64, x0:x0 + 64].clone() for f, y0, x0 in CROPS]
    torch.save({"cfg": cfg, "T": T, "H": H, "W": W, "z_seed": 4321, "sub16": out[:, :, ::16, ::16].clone(), "crops": crops,
                "crop_pos": CROPS, "mean": out.mean(dim=(2, 3)), "sqmean": out.pow(2).mean(dim=(2, 3)),
                "norm": out.norm().item()}, os.path.join(GOLD, "vae_fullres.pt"))
    print(f"[vae fullres] reference decode {tuple(out.shape)} in {time.time() - t0:.0f} s", flush=True)


if __name__ == "__main__":
    want = sys.argv[1:] or ["unet_kubric", "unet_pardom", "traj25", "traj50", "vae_fullres"]
    torch.manual_seed(0)
    if "unet_kubric" in want:
        pin_unet_metric("kubric", O.UNET_KUBRIC)
    if "unet_pardom" in want:
        pin_unet_metric("pardom", O.UNET_PARDOM)
    if "traj50" in want:
        pin_traj("traj50", O.UNET_KUBRIC, 14, 16, 24, 50, 2.5, keep=(1, 10, 25, 50))
    if "traj25" in want:
        pin_traj("traj25", O.UNET_KUBRIC, 14, 32, 48, 25, 1.5, keep=(1, 5, 10, 25), w_stride=2)
    if "vae_fullres" in want:
        pin_decoder_fullres()
