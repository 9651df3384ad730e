"""`gcd_frame_metrics` (PSNR / SSIM, full and masked) on flat, near-flat and 8-bit content against the oracle pinned to the
reference's `masked_ssim` (float32 images, scipy window means) and against the same formula in float64.

In a flat window the variance `uxx - ux*ux` is a difference of two nearly equal window means divided by C2 = 9e-4, so any
rounding of those means that differs from scipy's shows up in SSIM almost undamped. The kernel forms the means the way
`uniform_filter` does (fp32 products, vertical pass then horizontal, each summed in fp64 and rounded to fp32 once), so it meets
the oracle except where scipy's running mean lands on the other side of an fp32 rounding point. The bound allows a few such
one-ulp flips per frame: with E the largest change of a window's S (in float64) when one of its five means moves by one fp32 ulp
and n the number of windows averaged per channel, |kernel - oracle| <= 1e-12 + 8 E / (3 n)."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.ndimage import binary_erosion, uniform_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metrics_oracle as M  # noqa: E402

pytestmark = pytest.mark.gpu

PAD = 3
FLIPS = 8                        # one-ulp flips of a window mean allowed per frame
PSNR_TOL = 1e-9                  # dB


def _ulp_sensitivity(means32):
    """E: max over the given windows and over the five means of |S(mean +- 1 ulp) - S|, in float64 from the oracle's float32
    means (a list of five equally shaped float32 arrays)."""
    if means32[0].size == 0:
        return 0.0
    means = [m.astype(np.float64) for m in means32]
    s0 = M.ssim_map(*means)
    E = 0.0
    for k in range(5):
        for to in (np.float32(np.inf), np.float32(-np.inf)):
            p = list(means)
            p[k] = np.nextafter(means32[k], to).astype(np.float64)
            E = max(E, float(np.abs(M.ssim_map(*p) - s0).max()))
    return E


def _eroded(mask):
    return binary_erosion(mask, iterations=PAD)[PAD:-PAD, PAD:-PAD]


def _frame_bounds(p, g, keep):
    """E over the three channels of one frame for the whole cropped map and for the windows `keep` selects."""
    ms = [[m[PAD:-PAD, PAD:-PAD] for m in M.window_means(p[c], g[c])] for c in range(3)]
    E_all = max(_ulp_sensitivity(m) for m in ms)
    E_keep = max(_ulp_sensitivity([v[keep] for v in m]) for m in ms) if keep is not None else None
    return E_all, E_keep


def _run(pred, gt, mask):
    from gcd_b200 import metrics
    r = metrics.frame_metrics(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(),
                              None if mask is None else torch.from_numpy(mask).cuda())
    return {k: v.numpy() for k, v in r.items()}


def _check_psnr(got, p, g, sel=None):
    if sel is not None:
        mb = np.broadcast_to(sel, p.shape)
        if not mb.any():
            assert np.isnan(got)
            return
        p, g = p[mb], g[mb]
    want = M.psnr_skimage(p, g)
    if np.isinf(want):
        assert np.isinf(got) and got > 0, (got, want)
    else:
        assert abs(got - want) <= PSNR_TOL, (got, want)


# ---------------------------------------------------------------------------------------------------------------- content families
def _levels(rng, n):
    """Non-dyadic flat levels per frame and channel."""
    return rng.choice(np.array([0.93, 0.41, 0.17, 0.7, 0.3, 0.55, 0.06, 0.81], np.float32), size=(n, 3, 1, 1))


def _blocks(rng, n, H, W, b=32):
    lv = rng.integers(0, 256, size=(n, 3, (H + b - 1) // b, (W + b - 1) // b)).astype(np.float32) / np.float32(255)
    return np.repeat(np.repeat(lv, b, axis=2), b, axis=3)[:, :, :H, :W]


def _kubric(n, H, W):
    g = torch.load(os.path.join(ROOT, "tests", "golden", "render_kubric.pt"))
    f = ((g["rgb_dst"] + 1) / 2).clamp(0, 1).numpy().astype(np.float32)            # (3 frames, 3, 48, 72)
    f = f[np.arange(n) % f.shape[0]]
    reps = (1, 1, -(-H // f.shape[2]), -(-W // f.shape[3]))
    return np.ascontiguousarray(np.tile(f, reps)[:, :, :H, :W])


def _step(rng, shape):
    return rng.choice(np.array([-1, 1], np.float32), size=shape) / np.float32(255)


def family(name, n, H, W, seed):
    """(pred, gt) float32 (n, 3, H, W) in [0, 1]."""
    rng = np.random.default_rng(seed)
    sh = (n, 3, H, W)
    if name == "flat":                               # gt flat at a non-dyadic level, pred one 8-bit step away
        gt = np.broadcast_to(_levels(rng, n), sh).copy()
        pred = gt + _step(rng, (n, 3, 1, 1))
    elif name == "near_flat":                        # both sigma = 1e-3 around a level
        c = _levels(rng, n)
        gt = c + np.float32(1e-3) * rng.standard_normal(sh, dtype=np.float32)
        pred = c + np.float32(1e-3) * rng.standard_normal(sh, dtype=np.float32)
    elif name == "ramp":                             # horizontal / vertical ramps + 2e-3 noise
        t = (np.arange(W, dtype=np.float32) / np.float32(W))[None, None, None, :]
        v = (np.arange(H, dtype=np.float32) / np.float32(H))[None, None, :, None]
        gt = np.float32(0.2) + np.float32(0.5) * np.where(np.arange(n)[:, None, None, None] % 2 == 0, t, v)
        gt = np.broadcast_to(gt, sh).astype(np.float32)
        pred = gt + np.float32(2e-3) * rng.standard_normal(sh, dtype=np.float32)
    elif name == "blocks8":                          # 32x32 blocks of 8-bit levels, pred +-1/255 per pixel
        gt = _blocks(rng, n, H, W)
        pred = gt + _step(rng, sh) * (rng.random(sh) < 0.5)
    elif name == "kubric":                           # rendered frames against a copy with 1/255 noise
        gt = _kubric(n, H, W)
        pred = gt + np.float32(1 / 255) * rng.standard_normal(sh, dtype=np.float32)
    elif name == "noise":                            # control: what the suite tested before
        gt = rng.random(sh, dtype=np.float32)
        pred = gt + np.float32(0.1) * rng.standard_normal(sh, dtype=np.float32)
    else:
        raise ValueError(name)
    return np.clip(pred, 0, 1).astype(np.float32), np.clip(gt, 0, 1).astype(np.float32)


def masks(H, W, seed):
    """Three masks per size: a rectangle touching three image borders, a region whose edges sit on the 32x16 tile borders with
    holes, and random blobs; plus one whose erosion is empty (a 5-pixel band) and one selecting a single pixel."""
    rng = np.random.default_rng(seed)
    m = np.zeros((5, H, W), bool)
    m[0, :, : max(W // 2, 1)] = True
    m[1, 16 % H: H - 16 % H if H > 32 else H, 0: min(64, W)] = True
    if H >= 14 and W >= 14:
        m[1, H // 2 - 1: H // 2 + 1, W // 2 - 1: W // 2 + 2] = False
        m[1, :, min(32, W - 1)] = False
    m[2] = rng.random((H, W)) > 0.03
    m[2, (np.arange(H)[:, None] // 8 + np.arange(W)[None, :] // 8) % 5 == 0] = False
    m[3, max(H // 2 - 2, 0): H // 2 + 3, :] = True
    m[4, H // 2, W // 2] = True
    return m


def _check_ssim(got, want, E, n, label):
    bound = 1e-12 + FLIPS * E / (3 * n)
    assert abs(got - want) <= bound, f"{label}: kernel {got!r} oracle {want!r} |d| {abs(got - want):.3e} bound {bound:.3e}"


def _check_not_above_one(got, want, label):
    """SSIM <= 1 up to rounding. The reference's float32 formula itself exceeds 1 where the window variances are pure rounding
    (in 7x7 windows of sigma = 1e-4 noise by up to 1.4e-4), so the kernel may exceed 1 only as far as the oracle does."""
    assert got <= max(want, 1.0) + 1e-7, f"{label}: kernel SSIM {got!r} > 1 (oracle {want!r})"


def _check_vs64(got, want, s64, label):
    assert abs(got - s64) <= abs(want - s64) + 1e-9, f"{label}: kernel {got!r} float64 {s64!r} oracle {want!r}"


# ---------------------------------------------------------------------------------------------------------------- (b) full frames
SIZES = [(7, 7), (16, 32), (17, 33), (22, 38), (45, 71), (256, 384), (576, 1024)]
FAMILIES = ["flat", "near_flat", "ramp", "blocks8", "kubric", "noise"]


@pytest.mark.parametrize("H,W", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
@pytest.mark.parametrize("fam", FAMILIES)
def test_frame_metrics_full_frames_vs_oracle(fam, H, W):
    masks_ = masks(H, W, seed=H * 1000 + W)
    nm = masks_.shape[0]
    pred, gt = family(fam, nm, H, W, seed=FAMILIES.index(fam) * 100003 + H * 1009 + W)
    r = _run(pred, gt, None)
    rm = _run(pred, gt, masks_)
    n_all = (H - 2 * PAD) * (W - 2 * PAD)
    for t in range(nm):
        p, g = pred[t], gt[t]
        want_all, want_m = M.ssim_pair(p, g, masks_[t])
        s64_all, s64_m = M.ssim_pair(p, g, masks_[t], dtype=np.float64)
        keep = _eroded(masks_[t])
        E_all, E_m = _frame_bounds(p, g, keep)
        label = f"{fam} {H}x{W} frame {t}"
        for got in (r["ssim"][t], rm["ssim"][t]):
            _check_ssim(got, want_all, E_all, n_all, label + " ssim")
            _check_vs64(got, want_all, s64_all, label + " ssim")
            _check_not_above_one(got, want_all, label)
        if not keep.any():
            assert np.isnan(want_m) and np.isnan(rm["ssim_masked"][t]), label
        else:
            _check_ssim(rm["ssim_masked"][t], want_m, E_m, int(keep.sum()), label + " ssim_masked")
            _check_vs64(rm["ssim_masked"][t], want_m, s64_m, label + " ssim_masked")
            _check_not_above_one(rm["ssim_masked"][t], want_m, label)
        _check_psnr(r["psnr"][t], p, g)
        _check_psnr(rm["psnr_masked"][t], p, g, masks_[t][None])
    # identical frames: SSIM exactly 1 (flat non-dyadic levels included) and PSNR +inf
    same = _run(gt, gt.copy(), masks_)
    assert (same["ssim"] == 1.0).all() and np.isposinf(same["psnr"]).all(), (same["ssim"], same["psnr"])
    nonempty = np.array([_eroded(m).any() for m in masks_])
    assert (same["ssim_masked"][nonempty] == 1.0).all() and np.isnan(same["ssim_masked"][~nonempty]).all()


def test_frame_metrics_psnr_one_ulp_and_single_pixel():
    """pred = gt + 1 ulp: a very large, finite PSNR; masks that select a single pixel."""
    H, W = 45, 71
    rng = np.random.default_rng(11)
    gt = np.concatenate([_blocks(rng, 2, H, W), np.broadcast_to(_levels(rng, 2), (2, 3, H, W))]).astype(np.float32)
    gt = np.clip(gt, np.float32(1 / 255), np.float32(254 / 255))
    pred = np.nextafter(gt, np.float32(2)).astype(np.float32)
    m = np.zeros((4, H, W), bool)
    m[0, 0, 0] = m[1, H - 1, W - 1] = m[2, 17, 33] = m[3, 20, 40] = True
    r = _run(pred, gt, m)
    for t in range(4):
        assert np.isfinite(r["psnr"][t]) and r["psnr"][t] > 120, r["psnr"][t]
        _check_psnr(r["psnr"][t], pred[t], gt[t])
        _check_psnr(r["psnr_masked"][t], pred[t], gt[t], m[t][None])
        assert np.isnan(r["ssim_masked"][t])


# ---------------------------------------------------------------------------------------------------------------- (a) one window
def one_window_frames(seed=7):
    """About 20 000 7x7 frames: exactly one SSIM window per channel. Returns pred, gt (N, 3, 7, 7) float32, mask (N, 7, 7)."""
    rng = np.random.default_rng(seed)
    P, G = [], []
    sh = (3, 7, 7)

    def add(p, g):
        P.append(np.clip(np.asarray(p, np.float32), 0, 1).astype(np.float32))
        G.append(np.clip(np.asarray(g, np.float32), 0, 1).astype(np.float32))

    one = np.float32(1 / 255)
    for k in range(256):                                                    # every 8-bit level, flat
        g = np.full(sh, np.float32(k) / np.float32(255), np.float32)
        for p in (g, g + one, g - one, np.nextafter(g, np.float32(2)), np.nextafter(g, np.float32(-1))):
            add(p, g)
    for s in (1e-4, 1e-3, 1e-2):                                            # level + Gaussian noise
        for _ in range(3000):
            c = np.float32(rng.integers(0, 256)) / np.float32(255) if rng.random() < 0.5 else rng.random(dtype=np.float32)
            add(c + np.float32(s) * rng.standard_normal(sh, dtype=np.float32), c + np.float32(s) * rng.standard_normal(sh, dtype=np.float32))
    for _ in range(4000):                                                   # random 8-bit levels
        g = rng.integers(0, 256, size=sh).astype(np.float32) / np.float32(255)
        add(g + _step(rng, sh) * (rng.random(sh) < 0.5), g)
    for _ in range(3000):                                                   # uniform [0, 1]
        add(rng.random(sh, dtype=np.float32), rng.random(sh, dtype=np.float32))
    for _ in range(1000):                                                   # exact 0 and 1
        add(rng.integers(0, 2, size=sh).astype(np.float32), rng.integers(0, 2, size=sh).astype(np.float32))
    for v in (0.0, 1.0):
        for w in (0.0, 1.0):
            add(np.full(sh, v), np.full(sh, w))
    for _ in range(1500):                                                   # pred = gt with its channels swapped
        g = rng.random(sh, dtype=np.float32) if rng.random() < 0.5 else rng.integers(0, 256, size=sh).astype(np.float32) / np.float32(255)
        add(g[[1, 2, 0]], g)
    pred, gt = np.stack(P), np.stack(G)
    N = pred.shape[0]
    yy, xx = np.mgrid[0:7, 0:7]
    diamond = np.abs(yy - 3) + np.abs(xx - 3) <= 3
    mask = np.zeros((N, 7, 7), bool)
    kind = rng.integers(0, 4, size=N)
    mask[kind == 0] = True                                                  # keeps the window
    mask[kind == 1] = diamond                                               # the smallest mask that keeps it
    for i in np.nonzero(kind == 2)[0]:                                      # the diamond less one pixel: drops it
        m = diamond.copy()
        ys, xs = np.nonzero(diamond)
        j = rng.integers(0, ys.size)
        m[ys[j], xs[j]] = False
        mask[i] = m
    mask[kind == 3] = rng.random((int((kind == 3).sum()), 7, 7)) > 0.1     # random: keeps it or not
    return pred, gt, mask


def test_frame_metrics_one_window_frames():
    pred, gt, mask = one_window_frames()
    N = pred.shape[0]
    assert 19000 <= N <= 21845
    r = _run(pred, gt, mask)
    # the centre window of every frame and channel, batched: uniform_filter skips the size-1 axes, so each 7x7 channel is
    # filtered exactly as on its own
    m32 = [uniform_filter(v, size=(1, 1, 7, 7))[:, :, 3, 3] for v in (pred, gt, pred * pred, gt * gt, pred * gt)]
    p64, g64 = pred.astype(np.float64), gt.astype(np.float64)
    s64 = M.ssim_map(*[uniform_filter(v, size=(1, 1, 7, 7))[:, :, 3, 3] for v in (p64, g64, p64 * p64, g64 * g64, p64 * g64)]).mean(1)
    exact, worst = 0, 0.0
    for t in range(N):
        p, g = pred[t], gt[t]
        want, want_m = M.ssim_pair(p, g, mask[t])
        got = r["ssim"][t]
        E = _ulp_sensitivity([m[t] for m in m32])
        d = abs(got - want)
        exact += d <= 4 * 2.0 ** -52
        worst = max(worst, d / (1e-12 + FLIPS * E / 3))
        _check_ssim(got, want, E, 1, f"one-window frame {t}")
        _check_vs64(got, want, s64[t], f"one-window frame {t}")
        _check_not_above_one(got, want, f"one-window frame {t}")
        if _eroded(mask[t]).any():
            assert r["ssim_masked"][t] == got, (t, r["ssim_masked"][t], got)
        else:
            assert np.isnan(want_m) and np.isnan(r["ssim_masked"][t]), t
        _check_psnr(r["psnr"][t], p, g)
        _check_psnr(r["psnr_masked"][t], p, g, mask[t][None])
    assert exact >= 0.999 * N, f"{N - exact} of {N} one-window frames differ from the oracle by more than 4 ulp (worst {worst:.3f} of the bound)"
    same = _run(gt, gt.copy(), None)
    assert (same["ssim"] == 1.0).all() and np.isposinf(same["psnr"]).all()
