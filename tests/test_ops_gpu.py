"""GPU parity tests of the individual C-ABI ops against float64 torch math on the same (16-bit rounded) inputs.

Two checks per output: the relative L2 error over the whole tensor (bars stated for fp16 outputs, scaled to the operand type by
EM.tol16), and the per-element bound of oracle/error_model.py, which also sees one wrong tile in a large tensor and holds the
results beyond fp16's range to IEEE rounding (exactly +-inf in fp16, finite in bf16)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import error_model as EM

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from gcd_b200 import ops as o
    o.lib()
    return o


def rnd(*shape, scale=1.0, dtype=None, seed=[0]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    t = torch.randn(*shape, generator=g) * scale
    return t.cuda() if dtype is None else t.to(dtype).cuda()


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def conv3x3_im2col(x, stride=1, pad01=False):
    """float64 im2col of a channels-last act [n, H, W, C] for a 3x3 conv (padding 1), columns (ky, kx, c) like the packed
    weights: [n*Ho*Wo, 9*C]."""
    n, H, W, C = x.shape
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    cols = [xp[:, ky:ky + H:stride, kx:kx + W:stride, :] for ky in range(3) for kx in range(3)]
    return torch.cat(cols, -1).reshape(-1, 9 * C)


def conv_t3_im2col(x):
    """float64 im2col of act [B, T, HW, C] for Conv3d (3,1,1) with padding (1,0,0), columns (kt, c): [B*T*HW, 3*C]."""
    B, T, HW, C = x.shape
    xp = F.pad(x.double(), (0, 0, 0, 0, 1, 1))
    return torch.cat([xp[:, kt:kt + T] for kt in range(3)], -1).reshape(-1, 3 * C)


@pytest.mark.parametrize("M,K,N", [(300, 320, 320), (128, 64, 1280), (1000, 1280, 192), (28, 1280, 640), (513, 960, 2560)])
@pytest.mark.parametrize("out_f32", [True, False])
def test_linear_plain(ops, M, K, N, out_f32):
    AD = ops.act_dtype()
    x, w = rnd(M, K, dtype=AD), rnd(N, K, scale=K ** -0.5, dtype=AD)
    bias = rnd(N)
    out = torch.empty(M, N, device="cuda", dtype=torch.float32 if out_f32 else AD)
    ops.linear(x, w, ops.make_ep(out, bias=bias))
    ref = x.double() @ w.double().t() + bias.double()
    assert relerr(out, ref) < (2e-5 if out_f32 else EM.tol16(1e-3, AD))
    EM.check(out, ref, EM.gemm_scale(x, w, bias), "gemm", f"linear {M}x{K}x{N}")


def test_linear_epilogue_full(ops):
    AD = ops.act_dtype()
    M, K, N = 700, 320, 320
    x, w = rnd(M, K, dtype=AD), rnd(N, K, scale=K ** -0.5, dtype=AD)
    bias, rv = rnd(N), rnd(7, N)
    r1, r2 = rnd(M, N), rnd(M, N, dtype=AD)
    out = torch.empty(M, N, device="cuda")
    ops.linear(x, w, ops.make_ep(out, bias=bias, rowvec=rv, rows_per_vec=100, res1=r1, a_res1=0.3, res2=r2, a_res2=0.6,
                                 a_acc=0.7, act=1))
    rvr = rv.repeat_interleave(100, 0)
    acc = x.double() @ w.double().t() + bias.double() + rvr.double()
    ref = 0.7 * F.silu(acc) + 0.3 * r1.double() + 0.6 * r2.double()
    assert relerr(out, ref) < 2e-5
    scale = 0.7 * EM.gemm_scale(x, w, bias, rvr) + 0.3 * r1.double().abs() + 0.6 * r2.double().abs()
    EM.check(out, ref, scale, "gemm", "linear SiLU + rowvec + 2 residuals")
    # in-place residual update (out aliases res1)
    h = r1.clone()
    ops.linear(x, w, ops.make_ep(h, bias=bias, res1=h))
    ref = x.double() @ w.double().t() + bias.double() + r1.double()
    assert relerr(h, ref) < 2e-5
    EM.check(h, ref, EM.gemm_scale(x, w, bias, r1), "gemm", "linear in-place residual")


def test_linear_geglu(ops):
    AD = ops.act_dtype()
    M, K, C4 = 384, 320, 1280
    x = rnd(M, K, dtype=AD)
    w = rnd(2 * C4, K, scale=K ** -0.5, dtype=AD)   # rows [0,C4) value, [C4, 2*C4) gate (attention.py:93)
    b = rnd(2 * C4)
    idx = torch.arange(2 * C4).view(2, C4 // 16, 16).permute(1, 0, 2).reshape(-1).cuda()   # 16 value / 16 gate blocks
    out = torch.empty(M, C4, device="cuda", dtype=AD)
    ops.linear(x, w[idx].contiguous(), ops.make_ep(out, bias=b[idx].contiguous(), geglu=True))
    ref, scale, approx = geglu_ref(x, w, b)
    assert relerr(out, ref) < EM.tol16(1.5e-3, AD)
    EM.check(out, ref, scale, "gemm", "linear GEGLU", approx=approx)


def geglu_ref(x, w, b):
    """value * gelu(gate) in float64 (w rows [0, C4) value, [C4, 2*C4) gate), its scale (the value and gate GEMM scales
    times the sensitivities |gelu(gate)| and |value| * max |gelu'| = 1.13 |value|), and the kernel's stated approximation
    error of the polynomial GELU (gcd_b200/csrc/common.cuh geglu: <= 1.05e-4 |v| max(|g|, 4))."""
    C4 = w.shape[0] // 2
    y = x.double() @ w.double().t() + b.double()
    s = EM.gemm_scale(x, w, b)
    v, g = y[:, :C4], y[:, C4:]
    scale = s[:, :C4] * F.gelu(g).abs() + 1.13 * v.abs() * s[:, C4:]
    return v * F.gelu(g), scale, 1.05e-4 * v.abs() * g.abs().clamp_min(4.0)


def test_linear_strided_small_n(ops):
    AD = ops.act_dtype()
    M, K = 257, 320
    big = rnd(M, 3 * K, dtype=AD)
    x = big[:, K:2 * K]                       # strided rows
    w = rnd(4, K, scale=K ** -0.5, dtype=AD)
    out = torch.zeros(M, 4, device="cuda")
    ops.linear(x, w, ops.make_ep(out))
    ref = x.double() @ w.double().t()
    assert relerr(out, ref) < 2e-5
    EM.check(out, ref, EM.gemm_scale(x, w), "gemm", "linear strided N=4")


@pytest.mark.parametrize("n,H,W,C,Co", [(3, 18, 32, 64, 128), (2, 9, 16, 128, 160), (2, 8, 128, 64, 64),
                                        (5, 4, 6, 192, 320), (28, 2, 2, 64, 320), (1, 36, 64, 320, 640)])
@pytest.mark.parametrize("stride", [1, 2])
def test_conv2d_3x3(ops, n, H, W, C, Co, stride):
    AD = ops.act_dtype()
    x = rnd(n, H, W, C, dtype=AD)
    w = rnd(Co, C, 3, 3, scale=(9 * C) ** -0.5, dtype=AD)
    bias = rnd(Co)
    wp = w.permute(0, 2, 3, 1).reshape(Co, 9 * C).contiguous()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.empty(n * Ho * Wo, Co, device="cuda")
    ops.conv2d_3x3(x, wp, ops.make_ep(out, bias=bias), stride=stride)
    a = conv3x3_im2col(x, stride)
    ref = a @ wp.double().t() + bias.double()
    assert relerr(out, ref) < 3e-5
    EM.check(out, ref, EM.gemm_scale(a, wp, bias), "gemm", f"conv3x3 {n}x{H}x{W}x{C}->{Co} s{stride}")


@pytest.mark.parametrize("n,H,W,C,res,f32out", [(3, 24, 64, 448, True, True), (2, 9, 40, 640, False, False), (5, 16, 128, 960, True, True)])
def test_conv2d_3x3_wide_tiles_n320(ops, n, H, W, C, res, f32out):
    """N = 320 with K = 9*C >= 3840: two 160-column tiles per row tile and long k-loops, incl. ragged M, fp32 residual +
    fused GroupNorm statistics and 16-bit output."""
    AD = ops.act_dtype()
    Co = 320
    x = rnd(n, H, W, C, dtype=AD)
    w = rnd(Co, C, 3, 3, scale=(9 * C) ** -0.5, dtype=AD)
    bias = rnd(Co)
    wp = w.permute(0, 2, 3, 1).reshape(Co, 9 * C).contiguous()
    rows = n * H * W
    r0 = rnd(rows, Co)
    out = r0.clone() if f32out else torch.empty(rows, Co, device="cuda", dtype=AD)
    st = torch.zeros(max(n, 64) * 64, device="cuda", dtype=torch.float64)
    ok = ops.conv2d_3x3(x, wp, ops.make_ep(out, bias=bias, res1=out if res else None, a_res1=0.5 if res else 1.0,
                                             gn_stats=(st, Co // 32, 32, H * W)))
    a = conv3x3_im2col(x)
    ref = a @ wp.double().t() + bias.double()
    scale = EM.gemm_scale(a, wp, bias)
    del a
    if res:
        ref, scale = ref + 0.5 * r0.double(), scale + 0.5 * r0.double().abs()
    assert relerr(out, ref) < (3e-5 if f32out else EM.tol16(1e-3, AD))
    EM.check(out, ref, scale, "gemm", f"conv3x3 N=320 {n}x{H}x{W}x{C}")
    if ok:
        v = out.double().view(n, H * W, 32, Co // 32)
        want = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).reshape(-1)
        assert torch.allclose(st[: n * 64], want, rtol=1e-5, atol=1e-2)


@pytest.mark.parametrize("B,T,HW,C,Co", [(2, 14, 144, 128, 128), (1, 14, 4, 64, 320), (2, 14, 512, 320, 320), (3, 5, 96, 64, 64)])
def test_conv_t3(ops, B, T, HW, C, Co):
    AD = ops.act_dtype()
    x = rnd(B, T, HW, C, dtype=AD)
    w = rnd(Co, C, 3, 1, 1, scale=(3 * C) ** -0.5, dtype=AD)
    bias = rnd(Co)
    wp = w[:, :, :, 0, 0].permute(0, 2, 1).reshape(Co, 3 * C).contiguous()
    out = torch.empty(B * T * HW, Co, device="cuda")
    ops.conv_t3(x, wp, ops.make_ep(out, bias=bias))
    ref = F.conv3d(x.double().permute(0, 3, 1, 2).unsqueeze(-1), w.double(), bias.double(), padding=(1, 0, 0))  # b c t hw 1
    ref = ref.squeeze(-1).permute(0, 2, 3, 1).reshape(B * T * HW, Co)
    assert relerr(out, ref) < 3e-5
    a = conv_t3_im2col(x)
    assert torch.allclose(a @ wp.double().t() + bias.double(), ref)      # the im2col matches the Conv3d
    EM.check(out, ref, EM.gemm_scale(a, wp, bias), "gemm", f"conv_t3 {B}x{T}x{HW}x{C}->{Co}")


def test_bmm_nt(ops):
    AD = ops.act_dtype()
    G, M, K, N = 3, 200, 512, 300
    a, b = rnd(G, M, K, dtype=AD), rnd(G, N, K, scale=K ** -0.5, dtype=AD)
    out = torch.empty(G * M, N, device="cuda")
    ops.bmm_nt(a, b, ops.make_ep(out))
    ref = torch.bmm(a.double(), b.double().transpose(1, 2)).reshape(G * M, N)
    assert relerr(out, ref) < 2e-5
    scale = torch.bmm(a.double().abs(), b.double().abs().transpose(1, 2)).reshape(G * M, N)
    EM.check(out, ref, scale, "gemm", "bmm_nt")


GN_SHAPES = [(4, 9216, 320, True), (2, 14 * 64, 640, True), (3, 100, 960, False), (2, 333, 128, True), (1, 50, 2560, True),
             (2, 77, 512, False)]


@pytest.mark.parametrize("n_img,rows,C,f32", GN_SHAPES)
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm(ops, n_img, rows, C, f32, silu):
    AD = ops.act_dtype()
    x = rnd(n_img * rows, C) * 2 + 0.5
    if not f32:
        x = x.to(AD)
    g, b = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty(n_img * rows, C, device="cuda", dtype=AD)
    stats = torch.empty(n_img * 64, device="cuda", dtype=torch.float64)
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, silu, out, stats)
    ref, scale = groupnorm_ref(x, n_img, rows, C, g, b, silu)
    assert relerr(out, ref) < EM.tol16(1e-3, AD)
    EM.check(out, ref, scale, "norm", f"groupnorm {n_img}x{rows}x{C} f32={f32} silu={silu}")


def groupnorm_ref(x, n_img, rows, C, g, b, silu, groups=32):
    """GroupNorm (+ SiLU) in float64 and its scale: the normalised magnitude |g| (|x| + |mean|) / std + |b| of each element."""
    xr = x.double().view(n_img, rows, groups, C // groups)
    mean = xr.mean((1, 3), keepdim=True)
    rstd = (xr.var((1, 3), unbiased=False, keepdim=True) + 1e-5).rsqrt()
    gg, bb = g.double().view(groups, C // groups), b.double().view(groups, C // groups)
    ref = (xr - mean) * rstd * gg + bb
    scale = (xr.abs() + mean.abs()) * rstd * gg.abs() + bb.abs()
    if silu:
        ref = F.silu(ref)
    return ref.reshape(n_img * rows, C), scale.reshape(n_img * rows, C)


# ---- GroupNorm on groups whose mean is large against their spread. GroupNorm derives the variance as sum(x^2)/n - mean^2
# from the (sum, sum of squares) its producers accumulate: both terms are about mean^2, so the sums must be accurate far
# beyond fp32 for the difference to be. The reference (GroupNorm32: F.group_norm on x.float(), Welford moments) has no such
# limit. Inputs: R + sigma z per group, with a per-channel spread of +-1 % of sigma.
def offset_tensor(rows, C, R, sigma, dtype=torch.float32, seed=[0]):
    """[rows, C] = R + sigma * z + (+-1 % of sigma per channel), generated on the device, in `dtype`."""
    seed[0] += 1
    g = torch.Generator(device="cuda").manual_seed(seed[0])
    x = torch.randn(rows, C, device="cuda", generator=g).mul_(sigma)
    x.add_(R + 0.01 * sigma * (2 * torch.rand(C, device="cuda", generator=g) - 1))
    return x if dtype == torch.float32 else x.to(dtype)


def large_mean_16(dtype):
    """(R, sigma) for a 16-bit tensor: R = 3e4 (the fp16 range holds R + 5 sigma) and sigma = 8 ulps at R, so the spread
    survives the rounding. |mean| / std is then ~234 in fp16 and ~29 in bf16."""
    R = 3e4
    return R, 8 * 2.0 ** (math.floor(math.log2(R)) - (10 if dtype == torch.float16 else 7))


def group_moments(x, n_img, rows, C, groups=32):
    """float64 mean and variance (two-pass, centred) per (image, group) of x [n_img*rows, C], in row chunks (a float64
    copy of the largest tensors would not fit)."""
    xv = x.view(n_img, rows, groups, C // groups)
    step = max(1, (1 << 24) // (n_img * C))
    s = torch.zeros(n_img, groups, dtype=torch.float64, device=x.device)
    for r in range(0, rows, step):
        s += xv[:, r:r + step].double().sum((1, 3))
    mean = s / (rows * (C // groups))
    q = torch.zeros_like(s)
    for r in range(0, rows, step):
        q += (xv[:, r:r + step].double() - mean[:, None, :, None]).square().sum((1, 3))
    return mean, q / (rows * (C // groups))


def check_group_stats(st, x, n_img, rows, C, name, groups=32):
    """The mean and variance GroupNorm derives from the statistics buffer (sum, sum of squares per (image, group); the
    variance as gcd_groupnorm_apply forms it) against float64 moments of x, the tensor the producer read or stored:
        |d mean| <= 2^-19 (|mean| + std),   |d var| <= 2^-18 std (|mean| + std),
    linear in |mean| / std like the per-element bound of the "norm" class (oracle/error_model.py). Prints both worst
    error/bound ratios and returns the float64 moments and |mean| / std per group."""
    mean, var = group_moments(x, n_img, rows, C, groups)
    cnt = rows * (C // groups)
    s = st[: n_img * groups * 2].view(n_img, groups, 2)
    km = s[..., 0] / cnt
    kv = s[..., 1] / cnt - km * km
    std = var.sqrt()
    rm = ((km - mean).abs() / (2.0 ** -19 * (mean.abs() + std))).max().item()
    rv = ((kv - var).abs() / (2.0 ** -18 * std * (mean.abs() + std))).max().item()
    print(f"error/bound {name} statistics: mean {rm:.3f}, variance {rv:.3f}")
    assert rm <= 1 and rv <= 1, f"{name}: statistics error/bound mean {rm:.3g}, variance {rv:.3g}"
    return mean, var, mean.abs() / std


def groupnorm_ref_rows(x, idx, rows, mean, var, g, b, silu, groups=32):
    """groupnorm_ref for the rows `idx` of x [n_img*rows, C], from float64 moments of the whole tensor."""
    C = x.shape[1]
    xr = x[idx].double().view(len(idx), groups, C // groups)
    img = idx // rows
    m, rstd = mean[img][:, :, None], (var[img][:, :, None] + 1e-5).rsqrt()
    gg, bb = g.double().view(groups, C // groups), b.double().view(groups, C // groups)
    ref = (xr - m) * rstd * gg + bb
    scale = (xr.abs() + m.abs()) * rstd * gg.abs() + bb.abs()
    if silu:
        ref = F.silu(ref)
    return ref.reshape(len(idx), C), scale.reshape(len(idx), C)


@pytest.mark.parametrize("n_img,rows,C", [s[:3] for s in GN_SHAPES])
@pytest.mark.parametrize("R", [1e2, 1e3, 1e4, "16-bit"])
def test_groupnorm_large_mean(ops, n_img, rows, C, R):
    """gcd_groupnorm_stats + apply on groups with |mean| / std = R (float32 input, std 1) or the largest a 16-bit input
    holds: the statistics, then the output with its own statistics pass and, with SiLU, from the same statistics."""
    AD = ops.act_dtype()
    (R, sigma), dt = (large_mean_16(AD), AD) if R == "16-bit" else ((R, 1.0), torch.float32)
    x = offset_tensor(n_img * rows, C, R, sigma, dt)
    g, b = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty(n_img * rows, C, device="cuda", dtype=AD)
    stats = torch.empty(n_img * 64, device="cuda", dtype=torch.float64)
    name = f"groupnorm {n_img}x{rows}x{C} {dt} R={R:g}"
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, False, out, stats)
    _, _, ratio = check_group_stats(stats, x, n_img, rows, C, name)
    assert ratio.min() > 0.5 * R / sigma, ratio.min()
    ref, scale = groupnorm_ref(x, n_img, rows, C, g, b, False)
    EM.check(out, ref, scale, "norm", name)
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, True, out, stats, have_stats=True)
    ref, scale = groupnorm_ref(x, n_img, rows, C, g, b, True)
    EM.check(out, ref, scale, "norm", name + " SiLU")


# The GroupNorm statistics images of the production forward, which give the statistics kernel the most rows per thread.
@pytest.mark.parametrize("n_img,rows,C", [(28, 9216, 320),            # UNet spatial GroupNorm (14 frames x CFG)
                                          (2, 14 * 9216, 320),        # UNet temporal: one image per clip of 14 frames
                                          (1, 14 * 576 * 1024, 128)])  # VAE decoder temporal GroupNorm at full resolution
@pytest.mark.parametrize("f32", [True, False])
def test_groupnorm_large_mean_production_images(ops, n_img, rows, C, f32):
    """Statistics over every row against float64; the outputs (without and with SiLU) on a strided sample of rows."""
    AD = ops.act_dtype()
    (R, sigma), dt = ((1e4, 1.0), torch.float32) if f32 else (large_mean_16(AD), AD)
    x = offset_tensor(n_img * rows, C, R, sigma, dt)
    g, b = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty(n_img * rows, C, device="cuda", dtype=AD)
    stats = torch.empty(n_img * 64, device="cuda", dtype=torch.float64)
    name = f"groupnorm {n_img}x{rows}x{C} {dt} R={R:g}"
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, False, out, stats)
    mean, var, ratio = check_group_stats(stats, x, n_img, rows, C, name)
    assert ratio.min() > 0.5 * R / sigma, ratio.min()
    idx = torch.cat([torch.arange(0, n_img * rows, n_img * rows // 16384 + 1, device="cuda"),
                     torch.tensor([n_img * rows - 1], device="cuda")])
    ref, scale = groupnorm_ref_rows(x, idx, rows, mean, var, g, b, False)
    EM.check(out[idx], ref, scale, "norm", name + " (row sample)")
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, True, out, stats, have_stats=True)
    ref, scale = groupnorm_ref_rows(x, idx, rows, mean, var, g, b, True)
    EM.check(out[idx], ref, scale, "norm", name + " SiLU (row sample)")


@pytest.mark.parametrize("f32", [True, False])
def test_groupnorm_beyond_fp16_range(ops, f32):
    """Inputs of magnitude 1e5 (16-bit inputs only where the type holds them) and a gain that takes part of the output past
    65504: fp16 stores the IEEE-rounded +-inf there, bf16 finite values within the bound."""
    AD = ops.act_dtype()
    if not f32 and AD == torch.float16:
        pytest.skip("fp16 cannot hold the 1e5 inputs")
    n_img, rows, C = 2, 300, 320
    x = rnd(n_img * rows, C) * 1e5 + 3e4
    if not f32:
        x = x.to(AD)
    g, b = rnd(C) * 2e4 + 3e4, rnd(C) * 1e3
    out = torch.empty(n_img * rows, C, device="cuda", dtype=AD)
    stats = torch.empty(n_img * 64, device="cuda", dtype=torch.float64)
    ops.groupnorm(x, n_img, rows, C, g, b, 1e-5, False, out, stats)
    ref, scale = groupnorm_ref(x, n_img, rows, C, g, b, False)
    assert (ref.abs() > 7e4).sum() > 100
    EM.check(out, ref, scale, "norm", f"groupnorm |x| 1e5 f32={f32}")


@pytest.mark.parametrize("rows,C", [(1000, 320), (77, 640), (4032, 1280)])
def test_layernorm(ops, rows, C):
    AD = ops.act_dtype()
    x = rnd(rows, C) * 3 + 1
    g, b = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty(rows, C, device="cuda", dtype=AD)
    ops.layernorm(x, g, b, out)
    ref, scale = layernorm_ref(x, g, b)
    assert relerr(out, ref) < EM.tol16(1e-3, AD)
    EM.check(out, ref, scale, "norm", f"layernorm {rows}x{C}")
    # with frame-indexed additive embedding and sum output
    T, per = 7, 11
    add = rnd(T, C)
    so = torch.empty_like(x)
    ops.layernorm(x, g, b, out, add=add, add_rows_per=per, add_mod=T, sum_out=so)
    idx = (torch.arange(rows, device="cuda") // per) % T
    xs = x + add[idx]
    assert torch.equal(so, xs)
    ref, scale = layernorm_ref(xs, g, b)
    assert relerr(out, ref) < EM.tol16(1e-3, AD)
    EM.check(out, ref, scale, "norm", f"layernorm {rows}x{C} + frame embedding")


def layernorm_ref(x, g, b, eps=1e-5):
    """LayerNorm over the last dim in float64 and its scale |g| (|x| + |mean|) / std + |b|."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = (xd.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
    return (xd - mean) * rstd * g.double() + b.double(), (xd.abs() + mean.abs()) * rstd * g.double().abs() + b.double().abs()


@pytest.mark.parametrize("C", [320, 640, 1280, 192, 512])
def test_layernorm_large_mean(ops, C):
    """Rows with |mean| / std = 1e4 (a control: LayerNorm is two-pass in fp32) through the specialised C = 320 / 640 / 1280
    kernels and the generic one, 16-bit and float32 outputs. `sum_out` without `add` receives the input itself."""
    rows = 1000
    x = offset_tensor(rows, C, 1e4, 1.0)
    xd = x.double()
    assert (xd.mean(-1).abs() / xd.std(-1, unbiased=False)).min() > 5e3
    g, b = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    out = torch.empty(rows, C, device="cuda", dtype=ops.act_dtype())
    so = torch.full_like(x, float("nan"))
    ops.layernorm(x, g, b, out, sum_out=so)
    assert torch.equal(so, x)
    ref, scale = layernorm_ref(x, g, b)
    EM.check(out, ref, scale, "norm", f"layernorm {rows}x{C} R=1e4")
    out32 = torch.empty(rows, C, device="cuda")
    ops.layernorm_f32(x, g, b, out32)
    EM.check(out32, ref, scale, "norm", f"layernorm_f32 {rows}x{C} R=1e4")


def test_layernorm_beyond_fp16_range(ops):
    """Inputs of magnitude 1e5 and a gain that takes part of the 16-bit output past 65504 (+-inf in fp16, finite in bf16)."""
    rows, C = 500, 640
    x = rnd(rows, C) * 1e5 - 2e4
    g, b = rnd(C) * 2e4 + 3e4, rnd(C) * 1e3
    out = torch.empty(rows, C, device="cuda", dtype=ops.act_dtype())
    ops.layernorm(x, g, b, out)
    ref, scale = layernorm_ref(x, g, b)
    assert (ref.abs() > 7e4).sum() > 100
    EM.check(out, ref, scale, "norm", "layernorm |x| 1e5")


def test_softmax_rows(ops):
    AD = ops.act_dtype()
    x = rnd(300, 9216) * 5
    out = torch.empty(300, 9216, device="cuda", dtype=AD)
    ops.softmax_rows(x, 0.044, out)
    arg = (x.double() - x.double().amax(-1, keepdim=True)) * 0.044
    ref = torch.softmax(arg, -1)
    assert relerr(out, ref) < EM.tol16(2e-3, AD)
    EM.check(out, ref, ref * (1 + arg.abs()), "elementwise", "softmax_rows")   # exp's argument carries its own rounding


@pytest.mark.parametrize("clips,T,tokens,heads", [(2, 14, 144, 5), (1, 14, 37, 20), (1, 25, 16, 5)])
def test_attention_temporal(ops, clips, T, tokens, heads):
    AD = ops.act_dtype()
    C = heads * 64
    qkv = rnd(clips * T, tokens, 3 * C, dtype=AD)
    out = torch.empty(clips * T, tokens, C, device="cuda", dtype=AD)
    ops.attention_temporal(qkv, clips, T, tokens, heads, out)
    q, k, v = qkv.double().view(clips, T, tokens, 3, heads, 64).permute(3, 0, 2, 4, 1, 5)  # [clips, tokens, heads, T, 64]
    p = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1)                                 # over T
    ref = (p @ v).permute(0, 3, 1, 2, 4).reshape(clips * T, tokens, C)
    pv = (p @ v.abs()).permute(0, 3, 1, 2, 4).reshape(clips * T, tokens, C)
    assert relerr(out, ref) < EM.tol16(2e-3, AD)
    EM.check(out, ref, EM.attention_scale(pv, AD), "attention", f"attention_temporal {clips}x{T}x{tokens}x{heads}")


def test_elementwise(ops):
    AD = ops.act_dtype()
    x = rnd(2, 3, 5, 64)
    o = torch.empty(2, 6, 10, 64, device="cuda", dtype=AD)
    ops.upsample2x_to_act(x, 2, 3, 5, 64, o)
    ref = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(o, ref.to(AD))
    a, b = rnd(33, 64), rnd(33, 128)
    c = torch.empty(33, 192, device="cuda")
    ops.concat_channels(a, b, c)
    assert torch.equal(c, torch.cat([a, b], 1))
    t = torch.tensor([0.5756, -1.2, 3.0], device="cuda")
    e = torch.empty(3, 320, device="cuda")
    ops.timestep_embedding(t, 320, out_f32=e)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half).cuda()
    args = t[:, None] * freqs[None]
    assert (e - torch.cat([args.cos(), args.sin()], -1)).abs().max() < 2e-6


def test_sampler_kernels(ops):
    AD = ops.act_dtype()
    BT, T, H, W = 6, 3, 8, 16
    x, cc = rnd(BT, 4, H, W) * 10, rnd(BT, 4, H, W)
    sigma, sigma_next = 7.3, 5.1
    c_in = 1 / (sigma ** 2 + 1) ** 0.5
    buf = torch.empty(2 * BT, H, W, 64, device="cuda", dtype=AD)
    ops.sampler_prep(x, None, cc, BT, H, W, c_in, buf)
    ref = torch.zeros(2 * BT, 64, H, W, device="cuda")
    ref[:BT, :4] = x * c_in
    ref[BT:, :4] = x * c_in
    ref[BT:, 4:8] = cc
    assert torch.equal(buf, ref.permute(0, 2, 3, 1).to(AD))
    net = rnd(2 * BT, H, W, 16)
    scale = torch.linspace(1.0, 1.5, T).cuda()
    c_skip, c_out = 1 / (sigma ** 2 + 1), -sigma / (sigma ** 2 + 1) ** 0.5
    xn = x.clone()
    ops.sampler_update(xn, net, 16, BT, T, H, W, c_out, c_skip, sigma, sigma_next - sigma, scale)
    n4 = net[..., :4].permute(0, 3, 1, 2)
    den = n4 * c_out + torch.cat([x, x]) * c_skip
    du, dc = den[:BT], den[BT:]
    sc = scale.repeat(BT // T).view(BT, 1, 1, 1)
    d = du + sc * (dc - du)
    ref = x + (sigma_next - sigma) * (x - d) / sigma
    assert (xn - ref).abs().max() < 1e-4 * ref.abs().max()


def test_sampler_prep_beyond_fp16_range(ops):
    """c_in * x and the concat frames at magnitude 1e5: the IEEE-rounded 16-bit values (+-inf in fp16, finite in bf16)."""
    AD = ops.act_dtype()
    BT, H, W = 4, 8, 16
    x, cc = rnd(BT, 4, H, W) * 3e5, rnd(BT, 4, H, W) * 1e5
    c_in = 0.7
    buf = torch.empty(2 * BT, H, W, 64, device="cuda", dtype=AD)
    ops.sampler_prep(x, None, cc, BT, H, W, c_in, buf)
    exact = torch.zeros(2 * BT, 64, H, W, device="cuda")                 # the fp32 arithmetic of the kernel, then rounded
    exact[:BT, :4] = exact[BT:, :4] = x * c_in
    exact[BT:, 4:8] = cc
    assert torch.equal(buf, exact.permute(0, 2, 3, 1).to(AD))
    ref = torch.zeros(2 * BT, 64, H, W, device="cuda", dtype=torch.float64)
    ref[:BT, :4] = ref[BT:, :4] = x.double() * c_in
    ref[BT:, 4:8] = cc.double()
    ref = ref.permute(0, 2, 3, 1)
    assert (ref.abs() > 7e4).sum() > 100
    EM.check(buf, ref, ref.abs(), "elementwise", "sampler_prep |x| 1e5")


@pytest.mark.parametrize("case", ["linear", "linear_res", "conv"])
def test_gemm_beyond_fp16_range(ops, case):
    """GEMM / conv results and an fp32 residual of magnitude ~1e5 stored as 16-bit: exactly +-inf where the fp16 rounding of
    the result overflows (cooperative schedule without, ping-pong with the residual), finite values within the bound in bf16."""
    AD = ops.act_dtype()
    if case == "conv":
        n, H, W, C, Co = 2, 12, 16, 64, 128
        x = rnd(n, H, W, C, scale=300.0, dtype=AD)
        wp = rnd(Co, 9 * C, scale=300.0 * (9 * C) ** -0.5, dtype=AD)
        bias = rnd(Co) * 1e4
        out = torch.empty(n * H * W, Co, device="cuda", dtype=AD)
        ops.conv2d_3x3(x, wp, ops.make_ep(out, bias=bias))
        a = conv3x3_im2col(x)
        ref, scale = a @ wp.double().t() + bias.double(), EM.gemm_scale(a, wp, bias)
    else:
        M, K, N = 333, 256, 384
        x, w = rnd(M, K, scale=300.0, dtype=AD), rnd(N, K, scale=300.0 * K ** -0.5, dtype=AD)
        bias = rnd(N) * 1e4
        out = torch.empty(M, N, device="cuda", dtype=AD)
        r1 = rnd(M, N) * 1e5 if case == "linear_res" else None
        ops.linear(x, w, ops.make_ep(out, bias=bias, res1=r1, a_res1=0.5))
        ref, scale = x.double() @ w.double().t() + bias.double(), EM.gemm_scale(x, w, bias)
        if r1 is not None:
            ref, scale = ref + 0.5 * r1.double(), scale + 0.5 * r1.double().abs()
    assert (ref.abs() > 7e4).sum() > 100 and (ref.abs() < 6e4).sum() > 100
    EM.check(out, ref, scale, "gemm", f"{case} |y| ~1e5")


def _attn_ref(qkv, frames, tokens, heads):
    """softmax(q k^T / 8) v in float64, chunked over queries (attention.py:332-336 semantics), and sum_j p_j |v_j|."""
    C = heads * 64
    q, k, v = qkv.double().view(frames, tokens, 3, heads, 64).permute(2, 0, 3, 1, 4)
    outs, pvs = [], []
    for i in range(0, tokens, 2048):
        p = torch.softmax(torch.matmul(q[:, :, i:i + 2048], k.transpose(-1, -2)) * 0.125, -1)
        outs.append(torch.matmul(p, v))
        pvs.append(torch.matmul(p, v.abs()))
    cat = lambda ts: torch.cat(ts, 2).permute(0, 2, 1, 3).reshape(frames, tokens, C)
    return cat(outs), cat(pvs)


# 4096 / 9216 tokens: the level-1 shape bench.py runs at latent 72x128; 4100: ragged last key block; scale 6: logits ~ +-100,
# the running maximum moves by large steps from key block to key block (the kernel rescales on every block).
@pytest.mark.parametrize("frames,tokens,heads,scale", [
    (2, 256, 5, 1.5), (3, 144, 20, 1.5), (1, 576, 10, 1.5), (2, 100, 5, 1.5), (1, 2304, 5, 1.5), (2, 4, 5, 1.5),
    (2, 4096, 5, 1.5), (2, 9216, 5, 1.5), (1, 4100, 5, 1.5), (1, 9216, 5, 6.0), (1, 2304, 10, 6.0)])
def test_attention_spatial(ops, frames, tokens, heads, scale):
    AD = ops.act_dtype()
    C = heads * 64
    qkv = rnd(frames, tokens, 3 * C, dtype=AD, scale=scale)
    out = torch.empty(frames, tokens, C, device="cuda", dtype=AD)
    ops.attention_spatial(qkv, frames, tokens, heads, out)
    ref, pv = _attn_ref(qkv, frames, tokens, heads)
    assert relerr(out, ref) < EM.tol16(3e-3, AD)
    EM.check(out, ref, EM.attention_scale(pv, AD), "attention", f"attention_spatial {frames}x{tokens}x{heads} scale {scale}")


@pytest.mark.parametrize("n_img,Co,temporal", [(2, 128, False), (1, 128, True), (1, 512, False)])
def test_fused_groupnorm_stats_accumulated(ops, n_img, Co, temporal):
    """Images spanning >= 4 x num_SMs tiles take the per-CTA accumulation path (smem table, flush on image change) —
    the shape class of the VAE decoder's full-resolution convolutions (one clip or 14 frames over 64 512 tiles)."""
    AD = ops.act_dtype()
    C = 64
    if temporal:                                   # Conv3d (3,1,1) over [B=1, T=4, HW, C]; statistics over the whole clip
        T, HW = 4, 48 * 512
        x = rnd(1, T, HW, C, dtype=AD)
        wp = rnd(Co, 3 * C, scale=(3 * C) ** -0.5, dtype=AD)
        rows, rpi = T * HW, T * HW
        run = lambda ep: ops.conv_t3(x, wp, ep)
    else:
        H, W = (192, 512) if n_img == 2 else (256, 512)
        x = rnd(n_img, H, W, C, dtype=AD)
        wp = rnd(Co, 9 * C, scale=(9 * C) ** -0.5, dtype=AD)
        rows, rpi = n_img * H * W, H * W
        run = lambda ep: ops.conv2d_3x3(x, wp, ep)
    assert rpi // 128 >= 4 * torch.cuda.get_device_properties(0).multi_processor_count
    out = torch.empty(rows, Co, device="cuda", dtype=AD)
    st = torch.zeros(n_img * 64, device="cuda", dtype=torch.float64)
    assert run(ops.make_ep(out, bias=rnd(Co), gn_stats=(st, Co // 32, 32, rpi)))
    v = out.double().view(n_img, rpi, 32, Co // 32)
    ref = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).reshape(-1)
    assert torch.allclose(st, ref, rtol=1e-6, atol=1e-2)
    st2 = torch.zeros_like(st)                     # order-insensitive fp64 accumulation: repeats bit-for-bit (to fp64 rounding)
    assert run(ops.make_ep(out, bias=rnd(Co) * 0 , gn_stats=(st2, Co // 32, 32, rpi)))


@pytest.mark.parametrize("out_f32", [True, False])
def test_fused_groupnorm_stats(ops, out_f32):
    """gcd_epilogue.gn_stats: the conv epilogue accumulates (sum, sumsq) per (image, group) of the values it stores."""
    AD = ops.act_dtype()
    n, H, W, C, Co = 3, 8, 128, 64, 320
    x = rnd(n, H, W, C, dtype=AD)
    w = rnd(Co, C, 3, 3, scale=(9 * C) ** -0.5, dtype=AD)
    wp = w.permute(0, 2, 3, 1).reshape(Co, 9 * C).contiguous()
    bias = rnd(Co)
    out = torch.empty(n * H * W, Co, device="cuda", dtype=torch.float32 if out_f32 else AD)
    st = torch.zeros(n * 32 * 2, device="cuda", dtype=torch.float64)
    ok = ops.conv2d_3x3(x, wp, ops.make_ep(out, bias=bias, gn_stats=(st, Co // 32, 32, H * W)))
    assert ok
    v = out.double().view(n, H * W, 32, Co // 32)
    ref = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).reshape(-1)
    assert torch.allclose(st, ref, rtol=1e-5, atol=1e-3)
    # consumer: GroupNorm with the fused statistics == GroupNorm with its own statistics pass
    g, b = rnd(Co) * 0.1 + 1, rnd(Co) * 0.1
    y1 = torch.empty(n * H * W, Co, device="cuda", dtype=AD)
    y2 = torch.empty_like(y1)
    ops.groupnorm(out, n, H * W, Co, g, b, 1e-5, True, y1, st, have_stats=True)
    ops.groupnorm(out, n, H * W, Co, g, b, 1e-5, True, y2, torch.empty(n * 64, device="cuda", dtype=torch.float64))
    assert relerr(y1, y2) < 1e-5
    # a tiling that cannot guarantee one image per tile reports "not produced" instead of wrong statistics
    x2 = rnd(4, 4, 6, 64, dtype=AD)
    out2 = torch.empty(4 * 4 * 6, Co, device="cuda")
    assert not ops.conv2d_3x3(x2, wp, ops.make_ep(out2, bias=bias, gn_stats=(st, Co // 32, 32, 24)))


def test_conditioner_embedders_vs_reference(ops):
    """SURVEY.md §8(f) rank 1: ConcatTimestepEmbedderND and SphericalEmbedder (one kernel each) vs the reference classes' outputs."""
    from gcd_b200.embedders import ConcatTimestepEmbedderND, SphericalEmbedder
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "embedders.pt"))
    emb = ConcatTimestepEmbedderND(256)
    for k in ("1", "2"):
        y = emb(gold["concat_x" + k].cuda())
        assert y.shape == gold["concat_y" + k].shape and y.dtype == torch.float32
        # arguments reach 127 * 1 = 127 rad: cosf/sinf of the device vs the host libm agree to a few ulp of the argument
        assert (y.cpu() - gold["concat_y" + k]).abs().max() < 2e-5
    sph = SphericalEmbedder(128)
    sph.load_state_dict({"proj.weight": gold["sph_w"], "proj.bias": gold["sph_b"]})
    sph = sph.cuda()
    y = sph(gold["sph_x"].cuda())
    assert y.shape == gold["sph_y"].shape
    assert (y.cpu() - gold["sph_y"]).abs().max() < 1e-5 * max(1.0, float(gold["sph_y"].abs().max()))
    assert sph(gold["sph_x"].cuda().view(2, 14, 3)).shape == (2, 14, 128)


@pytest.mark.parametrize("n,rows,Ca,Cb", [(28, 9216, 640, 320), (28, 9216, 320, 320), (28, 144, 1280, 1280), (3, 100, 64, 192)])
def test_concat_channels_with_fused_groupnorm_stats(ops, n, rows, Ca, Cb):
    """Skip concat of the UNet's output blocks: one pass writes cat(a, b) and the (image, group) sums for the next GroupNorm."""
    a, b = rnd(n * rows, Ca) + 0.3, rnd(n * rows, Cb) * 2.0
    out = torch.empty(n * rows, Ca + Cb, device="cuda")
    st = torch.zeros(max(n, 64) * 64, device="cuda", dtype=torch.float64)
    ops.concat_channels(a, b, out, stats=st, n_img=n)
    ref = torch.cat([a, b], 1)
    assert torch.equal(out, ref)
    v = ref.double().view(n, rows, 32, (Ca + Cb) // 32)
    want = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).reshape(-1)
    assert torch.allclose(st[: n * 64], want, rtol=2e-6, atol=1e-3)
    st2 = torch.zeros_like(st)
    ops.concat_channels(a, b, out, stats=st2, n_img=n)
    assert torch.equal(st, st2)                       # fixed summation order inside a block; fp64 atomics across blocks
    # consumer equivalence: GroupNorm with these statistics == GroupNorm with its own statistics pass
    g, be = rnd(Ca + Cb) * 0.1 + 1, rnd(Ca + Cb) * 0.1
    AD = ops.act_dtype()
    y1 = torch.empty(n * rows, Ca + Cb, device="cuda", dtype=AD)
    y2 = torch.empty_like(y1)
    ops.groupnorm(out, n, rows, Ca + Cb, g, be, 1e-5, True, y1, st, have_stats=True)
    ops.groupnorm(out, n, rows, Ca + Cb, g, be, 1e-5, True, y2, torch.empty_like(st))
    assert relerr(y1, y2) < 1e-5
    out2 = torch.empty_like(out)
    ops.concat_channels(a, b, out2)                   # plain variant unchanged
    assert torch.equal(out2, ref)
    # 16-bit-only concat (what the UNet's output ResBlocks consume): the rounded values, statistics of the fp32 inputs
    out16 = torch.empty(n * rows, Ca + Cb, device="cuda", dtype=AD)
    st3 = torch.zeros_like(st)
    ops.concat_channels(a, b, out16, stats=st3, n_img=n)
    assert torch.equal(out16, ref.to(AD)) and torch.equal(st3, st)


@pytest.mark.parametrize("n,rows,Ca,Cb", [(3, 100, 64, 192), (28, 144, 1280, 1280), (2, 9216, 640, 320)])
@pytest.mark.parametrize("where", ["a", "b", "both"])
@pytest.mark.parametrize("R", [1e2, 1e3, 1e4])
def test_concat_channels_large_mean(ops, n, rows, Ca, Cb, where, R):
    """gcd_concat_channels_stats[_act] with the offset R (std 1) in `a`, in `b` or in both: the statistics against float64
    over the concatenation, equal in both variants, and the GroupNorm (without and with SiLU) that consumes them."""
    C = Ca + Cb
    a = offset_tensor(n * rows, Ca, R if where != "b" else 0.0, 1.0)
    b = offset_tensor(n * rows, Cb, R if where != "a" else 0.0, 1.0)
    out = torch.empty(n * rows, C, device="cuda")
    st = torch.zeros(n * 64, device="cuda", dtype=torch.float64)
    ops.concat_channels(a, b, out, stats=st, n_img=n)
    assert torch.equal(out, torch.cat([a, b], 1))
    name = f"concat_stats {n}x{rows}x({Ca}+{Cb}) offset in {where} R={R:g}"
    _, _, ratio = check_group_stats(st, out, n, rows, C, name)
    assert ratio.max() > 0.5 * R, ratio.max()
    AD = ops.act_dtype()
    st16 = torch.zeros_like(st)
    ops.concat_channels(a, b, torch.empty(n * rows, C, device="cuda", dtype=AD), stats=st16, n_img=n)
    assert torch.equal(st16, st)                      # the 16-bit variant sums the same fp32 inputs in the same order
    g, be = rnd(C) * 0.1 + 1, rnd(C) * 0.1
    y = torch.empty(n * rows, C, device="cuda", dtype=AD)
    for silu in (False, True):
        ops.groupnorm(out, n, rows, C, g, be, 1e-5, silu, y, st, have_stats=True)
        ref, scale = groupnorm_ref(out, n, rows, C, g, be, silu)
        EM.check(y, ref, scale, "norm", name + (" SiLU" if silu else ""))
