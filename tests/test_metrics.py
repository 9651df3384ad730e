"""Evaluation-loop image metrics (SURVEY.md §8(f) rank 3): oracle pinned to the reference's `masked_ssim` (CPU), CUDA kernel vs
the oracle and the golden (GPU). The kernel follows the reference's float32 arithmetic, so it differs only where scipy's running
window mean rounds one fp32 ulp the other way: SSIM within the flip bound of test_metrics_flat_gpu.py (a few such windows per
frame), PSNR within 1e-9 dB."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden", "metrics.pt")
GOLD_FLAT = os.path.join(ROOT, "tests", "golden", "metrics_flat.pt")


def test_oracle_matches_reference_golden():
    from oracle import metrics_oracle as M
    g = torch.load(GOLD)
    for t in range(g["gt"].shape[0]):
        a, m = M.ssim_pair(g["pred"][t].numpy(), g["gt"][t].numpy(), g["mask"][t].numpy())
        assert abs(a - g["ssim_all"][t]) < 1e-12
        assert (np.isnan(m) and np.isnan(g["ssim_masked"][t])) or abs(m - g["ssim_masked"][t]) < 1e-12
        assert abs(M.psnr(g["pred"][t].numpy(), g["gt"][t].numpy()) - g["psnr"][t]) < 1e-12


def test_oracle_matches_reference_golden_flat():
    """Flat, near-flat and 8-bit frames, and 7x7 frames with one SSIM window per channel (oracle/pin_metrics.py)."""
    from oracle import metrics_oracle as M
    g = torch.load(GOLD_FLAT)
    for key in ("", "7"):
        P, G, Mk = g["pred" + key], g["gt" + key], g["mask" + key]
        for t in range(G.shape[0]):
            a, m = M.ssim_pair(P[t].numpy(), G[t].numpy(), Mk[t].numpy())
            assert abs(a - g["ssim_all" + key][t]) < 1e-12
            want = g["ssim_masked" + key][t]
            assert (np.isnan(m) and np.isnan(want)) or abs(m - want) < 1e-12


def _ssim_bound(p, g, keep=None):
    """1e-12 + 8 E / (3 n): eight windows whose window mean rounds one fp32 ulp away from scipy's (test_metrics_flat_gpu.py)."""
    import test_metrics_flat_gpu as F
    E_all, E_keep = F._frame_bounds(p, g, keep)
    n = (p.shape[1] - 6) * (p.shape[2] - 6) if keep is None else int(keep.sum())
    return 1e-12 + F.FLIPS * (E_all if keep is None else E_keep) / (3 * n)


@pytest.mark.gpu
def test_frame_metrics_kernel_vs_reference_golden_and_oracle():
    from scipy.ndimage import binary_erosion
    from gcd_b200 import metrics
    from oracle import metrics_oracle as M
    for path in (GOLD, GOLD_FLAT):
        g = torch.load(path)
        r = metrics.frame_metrics(g["pred"].cuda(), g["gt"].cuda(), g["mask"].cuda())
        for t in range(g["gt"].shape[0]):
            p, q, mk = g["pred"][t].numpy(), g["gt"][t].numpy(), g["mask"][t].numpy()
            keep = binary_erosion(mk, iterations=3)[3:-3, 3:-3]
            assert abs(r["ssim"][t].item() - g["ssim_all"][t]) <= _ssim_bound(p, q)
            assert abs(r["psnr"][t].item() - M.psnr_skimage(p, q)) < 1e-9
            if np.isnan(g["ssim_masked"][t]):
                assert torch.isnan(r["ssim_masked"][t])
            else:
                assert abs(r["ssim_masked"][t].item() - g["ssim_masked"][t]) <= _ssim_bound(p, q, keep)
    # ragged size (not a multiple of the 32x16 tile), masked PSNR, identical images -> SSIM 1 / PSNR inf
    gen = torch.Generator().manual_seed(5)
    a = torch.rand(2, 3, 45, 71, generator=gen)
    b = (a + 0.1 * torch.randn(2, 3, 45, 71, generator=gen)).clamp(0, 1)
    m = torch.zeros(2, 45, 71, dtype=torch.bool)
    m[0, 4:41, 6:66] = True; m[0, 20:22, 30:33] = False        # a region with a hole (erosion eats 3 pixels around it)
    m[1, :, :35] = True                                         # touches three image borders (erosion border_value = 0)
    from scipy.ndimage import binary_erosion
    r = metrics.frame_metrics(a.cuda(), b.cuda(), m.cuda())
    for t in range(2):
        sa, sm = M.ssim_pair(a[t].numpy(), b[t].numpy(), m[t].numpy())
        keep = binary_erosion(m[t].numpy(), iterations=3)[3:-3, 3:-3]
        assert abs(r["ssim"][t].item() - sa) <= _ssim_bound(a[t].numpy(), b[t].numpy())
        assert abs(r["ssim_masked"][t].item() - sm) <= _ssim_bound(a[t].numpy(), b[t].numpy(), keep)
        mb = m[t][None].expand(3, -1, -1)
        assert abs(r["psnr_masked"][t].item() - M.psnr_skimage(a[t][mb].numpy(), b[t][mb].numpy())) < 1e-9   # test.py:395-399
    r = metrics.frame_metrics(a.cuda(), a.cuda())
    assert torch.isinf(r["psnr"]).all() and (r["ssim"] == 1).all()


@pytest.mark.gpu
def test_calculate_metrics_matches_reference_aggregation():
    """scripts/test.py:346-496: per-sample means over frames (nanmean), visible / occluded split, diversity."""
    from scipy.ndimage import binary_erosion
    from gcd_b200 import metrics
    from oracle import metrics_oracle as M
    gen = torch.Generator().manual_seed(9)
    S, T, H, W = 2, 3, 40, 64
    gt = torch.rand(T, 3, H, W, generator=gen)
    rep = gt.clone()
    rep[:, :, :, 40:] = 0.0                                    # right part occluded in the re-projection
    rep[2] = 0.0                                               # one frame fully occluded: visible metrics are NaN there
    pred = (gt[None] + 0.05 * torch.randn(S, T, 3, H, W, generator=gen)).clamp(0, 1)
    out, unc = metrics.calculate_metrics(gt.cuda(), rep.cuda(), pred.cuda())
    occ = rep.abs().sum(1) <= 1e-7
    for s in range(S):
        ps = [M.psnr_skimage(pred[s, t].numpy(), gt[t].numpy()) for t in range(T)]
        ss = [M.ssim_pair(pred[s, t].numpy(), gt[t].numpy())[0] for t in range(T)]
        sv = [M.ssim_pair(pred[s, t].numpy(), gt[t].numpy(), (~occ[t]).numpy())[1] for t in range(T)]
        bs = np.mean([_ssim_bound(pred[s, t].numpy(), gt[t].numpy()) for t in range(T)])
        keeps = [binary_erosion((~occ[t]).numpy(), iterations=3)[3:-3, 3:-3] for t in range(T)]
        bv = np.mean([_ssim_bound(pred[s, t].numpy(), gt[t].numpy(), keeps[t]) for t in range(2)])
        assert abs(out["mean_psnr"][s].item() - np.mean(ps)) < 1e-9 and abs(out["mean_ssim"][s].item() - np.mean(ss)) <= bs
        assert abs(out["mean_ssim_vis"][s].item() - np.nanmean(sv)) <= bv and np.isnan(sv[2])
    ref_div = np.nanmean(np.nanmean(np.std(pred.numpy(), axis=0), axis=1), axis=(1, 2))
    assert np.allclose(out["frame_diversity"].numpy(), ref_div, atol=1e-6)
    assert unc.shape == (T, H, W)
