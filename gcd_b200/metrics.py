"""Evaluation-loop metrics on the device (SURVEY.md §8(f) rank 3, first slice): per-frame PSNR / SSIM of decoded frames against
ground truth, full-frame and over visible / occluded masks, per-frame LPIPS (gcd_b200.lpips), and the per-sample aggregation of
gcd-model/scripts/test.py:346-496 (`calculate_metrics`). The per-pixel work runs in ONE kernel (csrc/metrics.cu); the few
per-frame scalars are folded on the host with the reference's own nanmean logic. No CPU fallback for the image pass."""
import ctypes
import math

import torch

from . import ops
from ._lib import check


def frame_metrics(pred, gt, mask=None):
    """pred, gt: CUDA float32 [frames, 3, H, W] in [0, 1]; mask: optional CUDA bool / uint8 [frames, H, W].
    Returns dict of float64 CPU tensors [frames]: psnr, ssim (+ psnr_masked, ssim_masked; NaN where the mask selects nothing)."""
    ops._need_cuda(pred, gt, mask)
    assert pred.shape == gt.shape and pred.dim() == 4 and pred.shape[1] == 3
    n, _, H, W = pred.shape
    pred = pred.to(torch.float32).contiguous()
    gt = gt.to(torch.float32).contiguous()
    m8 = None
    if mask is not None:
        assert tuple(mask.shape) == (n, H, W)
        m8 = mask.to(torch.uint8).contiguous()
    out = torch.empty(n, 8, device=pred.device, dtype=torch.float64)
    with ops._timed("elem", 0.0, n * 3 * H * W * 8):
        check(ops.lib().gcd_frame_metrics(ops._p(pred), ops._p(gt), ops._p(m8), n, H, W, ops._p(out), ops._stream()), "frame_metrics")
    o = out.cpu()
    nan = torch.full((n,), float("nan"), dtype=torch.float64)

    def ratio(num, den):
        return torch.where(den > 0, num / den.clamp(min=1), nan)

    def psnr(sq, cnt):                                   # skimage.metrics.peak_signal_noise_ratio, data_range = 1
        mse = ratio(sq, cnt)
        return torch.where(mse > 0, -10.0 * torch.log10(mse.clamp(min=1e-300)), torch.where(mse == 0, torch.full_like(mse, math.inf), nan))

    res = {"psnr": psnr(o[:, 0], o[:, 1]), "ssim": ratio(o[:, 4], o[:, 5])}
    if mask is not None:
        res["psnr_masked"] = psnr(o[:, 2], o[:, 3])
        res["ssim_masked"] = ratio(o[:, 6], o[:, 7])
    return res


def frame_lpips(pred, gt, model):
    """Per-frame LPIPS of frames in [0, 1] (validation_step, models/diffusion.py:342: `lpips(gt * 2 - 1, pred * 2 - 1)`).
    pred: CUDA [T, 3, H, W] or [S, T, 3, H, W]; gt: CUDA [T, 3, H, W]; model: gcd_b200.lpips.LPIPS. Returns float64 CPU [T] or
    [S, T]. With S samples the ground truth's features are computed once, not S times."""
    if gt.dim() != 4 or pred.shape[-4:] != gt.shape or pred.dim() not in (4, 5):
        raise ValueError(f"frame_lpips: pred {tuple(pred.shape)} does not match gt {tuple(gt.shape)} ([T,3,H,W] or [S,T,3,H,W])")
    ops._need_cuda(pred, gt)
    d = model.layer_distances(pred.reshape(-1, *gt.shape[1:]).float() * 2.0 - 1.0, gt.float() * 2.0 - 1.0)
    return d.sum(0).cpu().view(pred.shape[:-3])


def validation_metrics(gt_video, sampled_video, model):
    """DiffusionEngine.validation_step's metrics (models/diffusion.py:317-362): the means over frames of per-frame LPIPS, PSNR and
    SSIM. gt_video, sampled_video: CUDA float32 [frames, 3, H, W] in [0, 1]. Returns {lpips, psnr, ssim} as floats."""
    lp = frame_lpips(sampled_video, gt_video, model)
    m = frame_metrics(sampled_video, gt_video)
    return {"lpips": lp.mean().item(), "psnr": m["psnr"].mean().item(), "ssim": m["ssim"].mean().item()}


def _sample_std(pred_samples_rgb):
    return pred_samples_rgb.float().std(dim=0, unbiased=False)              # np.std(axis=0): (T, 3, H, W)


def _diversity(std):
    unc = std.mean(dim=1)                                                   # then nanmean over channels: (T, H, W)
    frame_diversity = unc.mean(dim=(1, 2)).double().cpu()
    return unc, frame_diversity, frame_diversity.mean()


def sample_diversity(pred_samples_rgb):
    """The spread of S samples (infer.py:185-211 calculate_metrics, test.py:458-462): pred_samples_rgb [S, T, 3, H, W] on the
    device. Returns (uncertainty [T, H, W] on the device: the per-pixel std over samples averaged over channels, frame_diversity
    float64 CPU [T]: its per-frame mean, mean_diversity: their mean, a float64 CPU scalar)."""
    return _diversity(_sample_std(pred_samples_rgb))


def calculate_metrics(gt_rgb, reproject_rgb, pred_samples_rgb, lpips=None):
    """gcd-model/scripts/test.py:346-496 for device tensors. gt_rgb [T,3,H,W]; reproject_rgb [T,3,H,W] or None (occluded where
    the re-projected colour is ~0, test.py:366-368); pred_samples_rgb [S,T,3,H,W]. Returns the reference's metrics dict
    (numpy-compatible CPU tensors) with the same keys. With an LPIPS model (gcd_b200.lpips.LPIPS) the dict also holds
    frame_lpips (S, T) and mean_lpips (S)."""
    S = pred_samples_rgb.shape[0]
    vis = occ = None
    if reproject_rgb is not None:
        occ = reproject_rgb.abs().sum(dim=1) <= 1e-7
        vis = ~occ
    keys = ["frame_psnr", "frame_ssim"] + (["frame_psnr_vis", "frame_ssim_vis", "frame_psnr_occ", "frame_ssim_occ"] if vis is not None else [])
    acc = {k: [] for k in keys}
    for s in range(S):
        m = frame_metrics(pred_samples_rgb[s], gt_rgb, vis)
        acc["frame_psnr"].append(m["psnr"]); acc["frame_ssim"].append(m["ssim"])
        if vis is not None:
            acc["frame_psnr_vis"].append(m["psnr_masked"]); acc["frame_ssim_vis"].append(m["ssim_masked"])
            mo = frame_metrics(pred_samples_rgb[s], gt_rgb, occ)
            acc["frame_psnr_occ"].append(mo["psnr_masked"]); acc["frame_ssim_occ"].append(mo["ssim_masked"])
    out = {k: torch.stack(v) for k, v in acc.items()}                     # (S, T)
    for k in keys:
        out[k.replace("frame_", "mean_")] = torch.nanmean(out[k], dim=1)  # (S)
    std = _sample_std(pred_samples_rgb)
    unc, out["frame_diversity"], out["mean_diversity"] = _diversity(std)
    if lpips is not None:
        out["frame_lpips"] = frame_lpips(pred_samples_rgb, gt_rgb, lpips)
        out["mean_lpips"] = out["frame_lpips"].mean(dim=1)
    if vis is not None:                    # test.py:470-480: the per-sample std over the masked pixels of each frame
        for name, m in (("vis", vis), ("occ", occ)):
            num = (std.double() * m[:, None]).sum(dim=(1, 2, 3))
            den = 3.0 * m.sum(dim=(1, 2)).double()
            fd = torch.where(den > 0, num / den.clamp(min=1), torch.full_like(num, float("nan"))).cpu()
            out[f"frame_diversity_{name}"] = fd
            out[f"mean_diversity_{name}"] = torch.nanmean(fd)
    return out, unc
