"""CPU restatement of the evaluation-loop image metrics (TEST INFRASTRUCTURE — only tests may import this).

* PSNR: scikit-image 0.22.0 (`requirements_versions.txt:40`, not vendored in the reference)
  `skimage.metrics.peak_signal_noise_ratio(a, b, data_range=1)` = 10 log10(1 / mean((a-b)^2)). Its `mean_squared_error` takes the
  difference and squares it in float32 (the images' float type) and only the mean in float64: `psnr_skimage`. `psnr` is the
  same value with the difference squared in float64, the form tests/golden/metrics.pt records; the two differ by at most about
  3e-7 dB (the fp32 rounding of the squares, 2^-24 relative).
* SSIM: scikit-image 0.22.0 `structural_similarity(a, b, data_range=1, channel_axis=0)` with its defaults (7x7 uniform window,
  sample covariance, K1 = 0.01, K2 = 0.03, 3-pixel border cropped, mean over channels), which the reference itself restates in
  gcd-model/scripts/eval_utils.py:571-664 (`masked_ssim`: element [0] of its result is the scikit-image value, element [1] the
  mean over `binary_erosion(mask, iterations=3)`).
  Its window means come from `scipy.ndimage.uniform_filter` on float32 images: one 1-D pass per axis, axis 0 first, each a running
  mean kept in float64 and rounded to float32 once per pass; the rest of the formula is float32 numpy arithmetic, left to right.
Pinned: tests/golden/metrics.pt holds outputs of the REFERENCE's `masked_ssim` source executed in the build container
(oracle/pin_metrics.py; the four scikit-image helper functions it imports are one-liners supplied by the pin script)."""
import numpy as np
from scipy.ndimage import binary_erosion, uniform_filter


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2, dtype=np.float64)
    return 10.0 * np.log10(1.0 / mse)


def psnr_skimage(a, b):
    """PSNR in scikit-image's operation order: the float32 difference squared in float32, the mean in float64."""
    d = a.astype(np.float32) - b.astype(np.float32)
    mse = np.mean(d * d, dtype=np.float64)
    return 10.0 * np.log10(1.0 / mse)


def window_means(x, y, win=7, dtype=np.float32):
    """The five window means of one channel pair (ux, uy, uxx, uyy, uxy), in `dtype`, as structural_similarity forms them."""
    x, y = x.astype(dtype), y.astype(dtype)
    return tuple(uniform_filter(v, size=win) for v in (x, y, x * x, y * y, x * y))


def ssim_map(ux, uy, uxx, uyy, uxy, win=7, K1=0.01, K2=0.03):
    """The SSIM map from the window means, in their dtype and in numpy's operation order."""
    NP = win ** 2
    cov = NP / (NP - 1)
    vx, vy, vxy = cov * (uxx - ux * ux), cov * (uyy - uy * uy), cov * (uxy - ux * uy)
    C1, C2 = K1 ** 2, K2 ** 2
    return ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))


def ssim_pair(im1, im2, mask=None, win=7, K1=0.01, K2=0.03, dtype=np.float32):
    """im1, im2: (3, H, W) float32 in [0, 1]; mask: (H, W) bool or None. Returns (ssim_all, ssim_masked or nan).
    dtype=np.float64 gives the same formula on float64 images (a higher-precision yardstick, not the reference's value)."""
    res = []
    pad = (win - 1) // 2
    for ch in range(im1.shape[0]):
        S = ssim_map(*window_means(im1[ch], im2[ch], win, dtype), win=win, K1=K1, K2=K2)
        Sc = S[pad:-pad, pad:-pad]
        allv = np.mean(Sc, dtype=np.float64)
        mv = np.nan
        if mask is not None:
            mc = binary_erosion(mask.astype(bool), iterations=pad)[pad:-pad, pad:-pad]
            mv = np.mean(Sc[mc], dtype=np.float64) if mc.any() else np.nan
        res.append((allv, mv))
    return tuple(np.mean(res, axis=0))
