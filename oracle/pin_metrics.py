"""Pins oracle/metrics_oracle.py to the REFERENCE's own `masked_ssim` (gcd-model/scripts/eval_utils.py:571-664), executed in the
build container, and writes tests/golden/metrics.pt (smoothed noise) and tests/golden/metrics_flat.pt (flat, near-flat and 8-bit
frames at 72 x 104 plus a batch of 7 x 7 frames with one SSIM window each) (TEST INFRASTRUCTURE; needs the reference checkout).

`masked_ssim` imports four helpers from scikit-image (0.22.0 in the reference's requirements_versions.txt, not installed here):
`_supported_float_type`, `check_shape_equality`, `slice_at_axis`, `crop` — one-liners provided below as a stub `skimage` package;
the function body that runs is the reference's.
    python -m oracle.pin_metrics
"""
import ast
import functools
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metrics_oracle as M  # noqa: E402

REF = os.path.join(os.environ.get("GCD_REFERENCE", ""), "scripts", "eval_utils.py")


def _stub_skimage():
    sk = types.ModuleType("skimage"); sh = types.ModuleType("skimage._shared"); ut = types.ModuleType("skimage._shared.utils")
    uu = types.ModuleType("skimage.util"); ac = types.ModuleType("skimage.util.arraycrop")
    ut._supported_float_type = lambda dt: np.float32 if np.dtype(dt).itemsize <= 4 else np.float64      # skimage/_shared/utils.py
    ut.check_shape_equality = lambda *a: None
    ut.warn = lambda *a, **k: None
    ut.slice_at_axis = lambda sl, axis: (slice(None),) * axis + (sl,) + (Ellipsis,)
    ac.crop = lambda ar, w: ar[tuple(slice(w, -w) for _ in range(ar.ndim))]
    sh.utils = ut; sk._shared = sh; uu.arraycrop = ac; sk.util = uu
    for name, m in (("skimage", sk), ("skimage._shared", sh), ("skimage._shared.utils", ut), ("skimage.util", uu), ("skimage.util.arraycrop", ac)):
        sys.modules[name] = m


def ref_masked_ssim():
    _stub_skimage()
    tree = ast.parse(open(REF).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "masked_ssim"]
    assert len(fn) == 1
    ns = {"np": np, "functools": functools}
    exec(compile(ast.Module(body=fn, type_ignores=[]), REF, "exec"), ns)
    return ns["masked_ssim"]


if __name__ == "__main__":
    f = ref_masked_ssim()
    g = torch.Generator().manual_seed(2024)
    T, H, W = 3, 72, 104
    gt = torch.rand(T, 3, H, W, generator=g)
    gt = torch.nn.functional.avg_pool2d(gt, 5, 1, 2)                                   # smooth "image"
    pred = (gt + 0.08 * torch.randn(T, 3, H, W, generator=g)).clamp(0, 1)
    mask = torch.zeros(T, H, W, dtype=torch.bool)
    mask[0, 10:50, 20:90] = True; mask[1] = torch.rand(H, W, generator=g) > 0.02; mask[2, :, :] = False; mask[2, 30:33, 40:43] = True
    out = {"gt": gt, "pred": pred, "mask": mask, "ssim_all": [], "ssim_masked": [], "psnr": []}
    for t in range(T):
        r = f(pred[t].numpy(), gt[t].numpy(), mask[t].numpy())
        o = M.ssim_pair(pred[t].numpy(), gt[t].numpy(), mask[t].numpy())
        assert abs(r[0] - o[0]) < 1e-12 and (abs(r[1] - o[1]) < 1e-12 or (np.isnan(r[1]) and np.isnan(o[1]))), (r, o)
        out["ssim_all"].append(float(r[0])); out["ssim_masked"].append(float(r[1])); out["psnr"].append(float(M.psnr(pred[t].numpy(), gt[t].numpy())))
    torch.save(out, os.path.join(ROOT, "tests", "golden", "metrics.pt"))
    print("[metrics] oracle == reference masked_ssim (both results) on", T, "frames:", out["ssim_all"], out["ssim_masked"], out["psnr"])

    # flat and near-flat content, where SSIM is most sensitive to how the window means are rounded
    H, W = 72, 104
    lv = torch.tensor([0.93, 0.41, 0.17])[:, None, None]
    step = torch.tensor([1.0, -1.0, 1.0])[:, None, None] / 255
    flat = lv.expand(3, H, W).clone()
    near = lv + 1e-3 * torch.randn(3, H, W, generator=g)
    b8 = torch.randint(0, 256, (3, (H + 31) // 32, (W + 31) // 32), generator=g).float() / 255
    b8 = b8.repeat_interleave(32, 1).repeat_interleave(32, 2)[:, :H, :W]
    gt = torch.stack([flat, near, b8]).float()
    pred = torch.stack([flat + step, lv + 1e-3 * torch.randn(3, H, W, generator=g),
                        b8 + torch.randint(-1, 2, (3, H, W), generator=g) / 255]).clamp(0, 1).float()
    mask = torch.zeros(3, H, W, dtype=torch.bool)
    mask[0, :, :52] = True; mask[1, 8:64, 16:96] = True; mask[1, 30:34, 40:44] = False; mask[2] = torch.rand(H, W, generator=g) > 0.05
    # 7 x 7 frames: one window per channel (flat 8-bit levels +- 1/255, level + 1e-3 noise, random 8-bit levels)
    N = 64
    lev = torch.randint(0, 256, (N, 3, 1, 1), generator=g).float() / 255
    g7 = torch.cat([lev[:24].expand(24, 3, 7, 7), lev[24:48] + 1e-3 * torch.randn(24, 3, 7, 7, generator=g),
                    torch.randint(0, 256, (16, 3, 7, 7), generator=g).float() / 255]).clamp(0, 1).float()
    p7 = torch.cat([g7[:24] + torch.where(torch.rand(24, 3, 1, 1, generator=g) < 0.5, 1.0, -1.0) / 255,
                    lev[24:48] + 1e-3 * torch.randn(24, 3, 7, 7, generator=g),
                    g7[48:] + torch.randint(-1, 2, (16, 3, 7, 7), generator=g) / 255]).clamp(0, 1).float()
    m7 = torch.rand(N, 7, 7, generator=g) > 0.05
    flat_out = {"gt": gt, "pred": pred, "mask": mask, "gt7": g7, "pred7": p7, "mask7": m7}
    for key, (P, G, Mk) in (("", (pred, gt, mask)), ("7", (p7, g7, m7))):
        rows = [(f(P[t].numpy(), G[t].numpy(), Mk[t].numpy()), M.ssim_pair(P[t].numpy(), G[t].numpy(), Mk[t].numpy()))
                for t in range(P.shape[0])]
        for r, o in rows:
            assert abs(r[0] - o[0]) < 1e-12 and (abs(r[1] - o[1]) < 1e-12 or (np.isnan(r[1]) and np.isnan(o[1]))), (r, o)
        flat_out["ssim_all" + key] = [float(r[0]) for r, _ in rows]
        flat_out["ssim_masked" + key] = [float(r[1]) for r, _ in rows]
    torch.save(flat_out, os.path.join(ROOT, "tests", "golden", "metrics_flat.pt"))
    print("[metrics] oracle == reference masked_ssim on 3 flat / near-flat / 8-bit frames and", N, "one-window frames:",
          flat_out["ssim_all"], flat_out["ssim_masked"])
