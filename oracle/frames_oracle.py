"""float64 numpy restatement of infer.py's frame preparation (gcd-model/sgm/data/common.py:121-199 after decoding, then
scripts/infer.py:137): u8 / 255 in fp32, center_crop_numpy, cv2.resize(INTER_LINEAR) of the float32 image, `* 2 - 1` and
`(x + 1) / 2` in fp32. The resize follows OpenCV's float32 path (resize.cpp: fx = (float)((d + 0.5) * scale - 0.5), floor,
fraction 0 and index clamped at both borders, weights 1 - fx, fx in fp32); the two weighted sums are taken in float64 and
rounded to fp32 once, so the kernel (unfused fp32 sums) and cv2 (SIMD fp32, FMA where the build has it) each lie a couple of
fp32 ulps from it."""
import numpy as np

from gcd_b200.infer import crop_box   # the host's restatement of center_crop_numpy, pinned against the reference's own


def cv_taps(n_out, n_in):
    """cv2 INTER_LINEAR taps along one axis: (i0 int64 [n_out], i1, w0 float32, w1 float32)."""
    scale = n_in / n_out
    fx = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    f = (fx - sx.astype(np.float32)).astype(np.float32)
    lo, hi = sx < 0, sx >= n_in - 1
    sx[lo], f[lo] = 0, 0
    sx[hi], f[hi] = n_in - 1, 0
    return sx, np.minimum(sx + 1, n_in - 1), (np.float32(1) - f).astype(np.float32), f


def resize_linear(img, hw):
    """img: float32 [H, W, C]; returns float32 [h, w, C] (float64 sums of the fp32-weighted taps, rounded once)."""
    H, W = img.shape[:2]
    h, w = hw
    if (H, W) == (h, w):
        return img.astype(np.float32)
    y0, y1, a0, a1 = cv_taps(h, H)
    x0, x1, b0, b1 = cv_taps(w, W)
    x = img.astype(np.float64)
    rows = x[:, x0] * b0[None, :, None].astype(np.float64) + x[:, x1] * b1[None, :, None].astype(np.float64)
    out = rows[y0] * a0[:, None, None].astype(np.float64) + rows[y1] * a1[:, None, None].astype(np.float64)
    return out.astype(np.float32)


def round_trip(p):
    """((p * 2 - 1) + 1) / 2 in fp32: process_image's output range and back, as infer.py computes input_rgb."""
    p = np.asarray(p, dtype=np.float32)
    return ((p * np.float32(2) - np.float32(1)) + np.float32(1)) / np.float32(2)


def prepare(frames, frame_hw, center_crop=True, channel_map=(0, 1, 2)):
    """frames: uint8 [n, H, W, C >= 3]. Returns float32 [n, 3, h, w] in [0, 1]: what gcd_frames_prepare computes."""
    frames = np.asarray(frames)
    rgb = frames[..., list(channel_map)].astype(np.float32) / np.float32(255)
    y0, x0, ch, cw = crop_box(frames.shape[1], frames.shape[2], frame_hw, center_crop)
    rgb = rgb[:, y0:y0 + ch, x0:x0 + cw]
    out = np.stack([resize_linear(f, frame_hw) for f in rgb])
    return round_trip(out).transpose(0, 3, 1, 2).copy()
