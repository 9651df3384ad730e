"""LPIPS on the H100: the CUDA path (gcd_b200.lpips: input stage, tc_gemm convs with the ReLU epilogue, max-pool, fused heads)
against the reference's goldens and the live fp32 oracle, its exact properties (zero distance to itself, symmetry, the shared ground
truth of [S, T] calls, run-to-run bits), its kernels in isolation, and the metrics built on it.

Tolerance (16-bit operands over 13 convolutions, fp32 accumulation): per-frame |LPIPS - fp32 oracle| and rel-L2 over all frames,
_tol(). Measured on one H100 80GB HBM3 (700 W) with the seeded weights of the goldens, distances 0.11..1.0:
  fp16 build: max |d| 2.6e-5, rel-L2 1.1e-4 (goldens); 6.2e-6 / 3.4e-5 (256x384); 4.4e-5 / 4.1e-5 (calculate_metrics);
              6.2e-5 / 2.7e-5 over one 28-frame evaluation example (tools/bench_lpips.py)  ->  bound 2e-4 / 1e-3;
  bf16 build: max |d| 1.8e-4, rel-L2 9.6e-4 (goldens); 1.2e-4 / 6.8e-4 (256x384); 2.7e-4 / 2.9e-4 (calculate_metrics)
              ->  bound 5e-4 / 2.5e-3."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _tol():
    from gcd_b200 import ops
    return (2e-4, 1e-3) if ops.act_dtype() == torch.float16 else (5e-4, 2.5e-3)


@pytest.fixture(scope="module")
def model():
    from gcd_b200.lpips import LPIPS
    from oracle import lpips_oracle as O
    g = torch.load(os.path.join(GOLD, "lpips.pt"))
    m = LPIPS()
    m.load_state_dict(O.seeded_state(g["meta"]["weight_seed"]))
    return m


@pytest.fixture(scope="module")
def sd_dev():
    from oracle import lpips_oracle as O
    g = torch.load(os.path.join(GOLD, "lpips.pt"))
    return {k: v.to(DEV) for k, v in O.seeded_state(g["meta"]["weight_seed"]).items()}


def _check(got, ref, what):
    got, ref = got.double().cpu().flatten(), ref.double().cpu().flatten()
    d = (got - ref).abs().max().item()
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"{what}: max |d| {d:.3e}  rel-L2 {rel:.3e}  (values {ref.min().item():.3f}..{ref.max().item():.3f})")
    abs_tol, rel_tol = _tol()
    assert d <= abs_tol and rel <= rel_tol, (what, d, rel)


def test_goldens(model):
    from oracle import lpips_oracle as O
    g = torch.load(os.path.join(GOLD, "lpips.pt"))
    for c, terms, val in zip(g["cases"], g["terms"], g["lpips"]):
        pred, gt = O.pair_inputs(c["n"], c["H"], c["W"], c["seed"])
        t = model.layer_distances(gt.to(DEV), pred.to(DEV))
        _check(t.sum(0), val, f"golden {c['H']}x{c['W']}")
        for k in range(5):
            assert (t[k].cpu() - terms[k].double()).abs().max().item() <= _tol()[0], k
        out = model(gt.to(DEV), pred.to(DEV))
        assert out.shape == (c["n"], 1, 1, 1) and out.dtype == torch.float32 and out.is_cuda


@pytest.mark.parametrize("H,W", [(256, 384), (90, 130)])
def test_live_oracle(model, sd_dev, H, W):
    from oracle import lpips_oracle as O
    pred, gt = O.pair_inputs(3, H, W, seed=H + W)
    pred, gt = pred.to(DEV), gt.to(DEV)
    with torch.no_grad():
        ref = O.lpips(sd_dev, gt, pred)
    _check(model(gt, pred).flatten(), ref, f"live oracle {H}x{W}")


def test_exact_properties(model):
    from oracle import lpips_oracle as O
    pred, gt = O.pair_inputs(4, 64, 96, seed=7)
    pred, gt = pred.to(DEV), gt.to(DEV)
    assert (model(gt, gt) == 0).all()                                         # LPIPS(x, x) == 0 exactly
    a = model(gt, pred)
    assert torch.equal(a, model(pred, gt))                                    # symmetric, bit for bit
    assert torch.equal(a, model(gt, pred))                                    # two runs, same bits
    assert (a > 0).all()


def test_shared_ground_truth_equals_per_sample_calls(model):
    from gcd_b200 import metrics
    from oracle import lpips_oracle as O
    S, T = 3, 5
    pred, gt = O.pair_inputs(S * T, 48, 80, seed=9)
    pred = ((pred.view(S, T, 3, 48, 80) + 1) / 2).to(DEV)
    gt = ((gt[:T] + 1) / 2).to(DEV)
    both = metrics.frame_lpips(pred, gt, model)
    assert both.shape == (S, T) and both.dtype == torch.float64 and not both.is_cuda
    for s in range(S):
        assert torch.equal(both[s], metrics.frame_lpips(pred[s], gt, model))


def test_chunked_frames_equal_one_chunk(model, monkeypatch):
    from gcd_b200 import lpips
    from oracle import lpips_oracle as O
    pred, gt = O.pair_inputs(6, 32, 48, seed=5)
    pred, gt = pred.to(DEV), gt.to(DEV)
    whole = model.layer_distances(pred, gt)
    monkeypatch.setattr(lpips, "ROWS_PER_CHUNK", 2 * 32 * 48)               # one (target, input) pair per chunk
    assert torch.equal(whole, model.layer_distances(pred, gt))


@pytest.mark.parametrize("C,N,H,W,f32", [(64, 64, 24, 40, False), (64, 128, 17, 33, False), (128, 256, 20, 24, False),
                                         (256, 512, 12, 20, False), (64, 64, 24, 40, True)])
def test_tc_gemm_relu_epilogue(C, N, H, W, f32):
    """act = 3 against relu of the act = 0 GEMM (bit for bit: rounding keeps the sign) and against float64 relu(conv).
    N = 64 runs on 128-wide tiles; the fp32 output takes the ping-pong schedule."""
    from gcd_b200 import ops
    AD = ops.act_dtype()
    g = torch.Generator().manual_seed(C + N)
    x = torch.randn(2, H, W, C, generator=g).to(AD).to(DEV)
    w = (torch.randn(N, 9 * C, generator=g) / (3 * C ** 0.5)).to(AD).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    od = torch.float32 if f32 else AD
    y3 = torch.empty(2 * H * W, N, device=DEV, dtype=od)
    y0 = torch.empty_like(y3)
    ops.conv2d_3x3(x, w, ops.make_ep(y3, bias=b, act=3))
    ops.conv2d_3x3(x, w, ops.make_ep(y0, bias=b))
    assert (y3.float() == torch.relu(y0.float())).all()
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().view(N, 3, 3, C).permute(0, 3, 1, 2), b.double(), padding=1)
    ref = torch.relu(ref).permute(0, 2, 3, 1).reshape(-1, N)
    tol = 2e-3 if AD == torch.float16 else 8e-3                              # one rounding of the 16-bit output
    assert ((y3.double() - ref).abs().max() / ref.abs().max()).item() < tol
    if not f32 and C == 64:                                                   # the 1-tap K = 64 form of conv1_1
        xl = x.view(-1, C)
        wl = w[:, :C].contiguous()
        yl = torch.empty(xl.shape[0], N, device=DEV, dtype=AD)
        ops.linear(xl, wl, ops.make_ep(yl, bias=b, act=3))
        rl = torch.relu(xl.double() @ wl.double().t() + b.double())
        assert ((yl.double() - rl).abs().max() / rl.abs().max()).item() < tol


@pytest.mark.parametrize("H,W", [(7, 9), (24, 40), (1, 5)])
def test_input_stage_against_unfold(H, W):
    from gcd_b200 import ops
    from gcd_b200.lpips import SCALE, SHIFT
    AD = ops.act_dtype()
    n = 2
    x = (torch.rand(n, 3, H, W, generator=torch.Generator().manual_seed(H * W)) * 2 - 1).to(DEV)
    shift, scale = torch.tensor(SHIFT, device=DEV), torch.tensor(SCALE, device=DEV)
    out = torch.full((n * H * W, 64), float("nan"), device=DEV, dtype=AD)
    ops.lpips_input(x, shift, scale, out)
    scaled = (x - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)
    u = F.unfold(scaled, 3, padding=1).view(n, 3, 3, 3, H * W)              # (c, ky, kx) x pixels; zeros outside the image
    ref = u.permute(0, 4, 2, 3, 1).reshape(n * H * W, 27)
    assert torch.equal(out[:, :27].float(), ref.to(AD).float())
    assert (out[:, 27:] == 0).all()


@pytest.mark.parametrize("H,W,C", [(7, 9, 64), (50, 70, 128), (3, 2, 512), (25, 35, 256)])
def test_maxpool_odd_sizes(H, W, C):
    from gcd_b200 import ops
    AD = ops.act_dtype()
    x = torch.randn(3, H, W, C, generator=torch.Generator().manual_seed(C)).to(AD).to(DEV)
    out = torch.empty(3, H // 2, W // 2, C, device=DEV, dtype=AD)
    ops.maxpool2x2(x, out)
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(out.float(), ref)


def test_head_against_torch():
    """One head launch against the normalised-difference formula in float64 on the same 16-bit features."""
    from gcd_b200 import ops
    AD = ops.act_dtype()
    g = torch.Generator().manual_seed(4)
    for C, HW in ((64, 3000), (512, 12), (256, 513)):
        feat = torch.relu(torch.randn(4, HW, C, generator=g)).to(AD).to(DEV)
        w = torch.rand(C, generator=g).to(DEV)
        pairs = torch.tensor([[0, 1], [2, 1], [3, 3]], dtype=torch.int32, device=DEV)
        out = torch.empty(3, device=DEV, dtype=torch.float64)
        partial = torch.full((3 * ((HW + ops.LPIPS_HEAD_PIX - 1) // ops.LPIPS_HEAD_PIX),), float("nan"), device=DEV, dtype=torch.float64)
        count = torch.zeros(3, device=DEV, dtype=torch.int32)
        ops.lpips_head(feat, pairs, w, partial, count, out)
        assert (count == 0).all()                                             # left ready for the next launch
        f = feat.double()
        nf = f / (f.norm(dim=2, keepdim=True) + 1e-10)
        ref = torch.stack([((nf[a] - nf[b]) ** 2 @ w.double()).mean() for a, b in pairs.tolist()])
        assert (out - ref).abs().max().item() < 1e-5 * ref.abs().max().item() + 1e-12
        assert out[2].item() == 0.0


def test_calculate_metrics_with_and_without_lpips(model, sd_dev):
    from gcd_b200 import metrics
    from oracle import lpips_oracle as O
    S, T, H, W = 2, 3, 64, 96
    pred, gt = O.pair_inputs(S * T, H, W, seed=21)
    pred = ((pred.view(S, T, 3, H, W) + 1) / 2).to(DEV)
    gt = ((gt[:T] + 1) / 2).to(DEV)
    rep = gt.clone()
    rep[:, :, :20] = 0
    for reproject in (None, rep):
        base, unc = metrics.calculate_metrics(gt, reproject, pred)
        full, unc2 = metrics.calculate_metrics(gt, reproject, pred, lpips=model)
        assert set(full) == set(base) | {"frame_lpips", "mean_lpips"}
        for k, v in base.items():       # frame_metrics sums blocks with fp64 atomics: equal up to their summation order
            torch.testing.assert_close(torch.as_tensor(full[k]), torch.as_tensor(v), rtol=1e-12, atol=0, equal_nan=True, msg=k)
        assert torch.equal(unc, unc2)
        with torch.no_grad():
            ref = torch.stack([O.lpips(sd_dev, gt * 2 - 1, pred[s] * 2 - 1) for s in range(S)])
        assert full["frame_lpips"].shape == (S, T) and full["mean_lpips"].shape == (S,)
        _check(full["frame_lpips"], ref, "calculate_metrics frame_lpips")
        assert torch.allclose(full["mean_lpips"], full["frame_lpips"].mean(1))


def test_validation_metrics(model, sd_dev):
    from gcd_b200 import metrics
    from oracle import lpips_oracle as O
    pred, gt = O.pair_inputs(4, 64, 96, seed=31)
    pred, gt = ((pred + 1) / 2).to(DEV), ((gt + 1) / 2).to(DEV)
    got = metrics.validation_metrics(gt, pred, model)
    assert set(got) == {"lpips", "psnr", "ssim"}
    with torch.no_grad():
        ref_lp = O.lpips(sd_dev, gt * 2 - 1, pred * 2 - 1).double().mean().item()
    fm = metrics.frame_metrics(pred, gt)
    assert abs(got["lpips"] - ref_lp) <= _tol()[0]
    # frame_metrics sums blocks with fp64 atomics: two calls agree up to that summation order
    assert got["psnr"] == pytest.approx(fm["psnr"].mean().item(), rel=1e-12)
    assert got["ssim"] == pytest.approx(fm["ssim"].mean().item(), rel=1e-12)
