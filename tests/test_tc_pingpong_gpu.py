"""GPU parity tests of tc_gemm's ping-pong schedule (ops with a residual or an fp32 output) at the edges of its 64-row tile geometry,
and of the cooperative 128-row schedule (plain 16-bit output) on the same problems: tile counts that leave one
consumer warpgroup without work or with one tile more than the other, k-step counts that do not divide the stage ring, and
fused GroupNorm statistics whose image boundary is a 64-row but not a 128-row boundary. Same references and error model as
test_ops_gpu.py: float64 torch math on the same (16-bit rounded) inputs, the relative L2 error and the per-element bound of
oracle/error_model.py."""
import pytest
import torch
import torch.nn.functional as F

from oracle import error_model as EM
from test_ops_gpu import check_group_stats, groupnorm_ref, large_mean_16, offset_tensor

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from gcd_b200 import ops as o
    o.lib()
    return o


def rnd(*shape, scale=1.0, dtype=None, seed=[1000]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    t = torch.randn(*shape, generator=g) * scale
    return t.cuda() if dtype is None else t.to(dtype).cuda()


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (M, K, N): M in 64-row tiles x N in 256 / 160 / 128-column tiles gives the tile count; with one CTA per SM a CTA runs
# ceil or floor of tiles / SMs of them, alternating between its two consumer warpgroups.
@pytest.mark.parametrize("M,K,N", [
    (64, 320, 256),                 # exactly one tile: the second warpgroup has none
    (3 * 64, 64, 256),              # odd tile count below the SM count; one k-step per tile
    (5 * 64 - 7, 5 * 64, 256),      # five k-steps with BN = 256 (five stages): every tile starts on stage 0
    (64 * 7, 7 * 64, 512),          # seven k-steps over five stages: tiles start on every stage, both ring phases
    (64 * 3, 3 * 64, 160),          # BN = 160 (eight stages), fewer k-steps than stages
    (64 * 5, 11 * 64, 128),         # BN = 128 (eight stages), more k-steps than stages
])
@pytest.mark.parametrize("out_f32", [True, False])
def test_linear_tile_edges(ops, M, K, N, out_f32):
    AD = ops.act_dtype()
    x, w = rnd(M, K, dtype=AD), rnd(N, K, scale=K ** -0.5, dtype=AD)
    bias = rnd(N)
    out = torch.empty(M, N, device="cuda", dtype=torch.float32 if out_f32 else AD)
    ops.linear(x, w, ops.make_ep(out, bias=bias))
    ref = x.double() @ w.double().t() + bias.double()
    assert relerr(out, ref) < (2e-5 if out_f32 else EM.tol16(1e-3, AD))
    EM.check(out, ref, EM.gemm_scale(x, w, bias), "gemm", f"linear {M}x{K}x{N}")


@pytest.mark.parametrize("extra", [1, 2])
def test_linear_odd_tiles_above_sm_count(ops, extra):
    """2 x SMs + 1 and 3 x SMs + 2 tiles: some CTAs run three tiles (two on warpgroup 0, one on warpgroup 1), with both
    residuals and the in-place update that the UNet's residual stream uses."""
    AD = ops.act_dtype()
    tiles = (1 + extra) * _sms() + extra
    M, K, N = tiles * 64 - 13, 192, 256
    x, w = rnd(M, K, dtype=AD), rnd(N, K, scale=K ** -0.5, dtype=AD)
    bias, r1, r2 = rnd(N), rnd(M, N), rnd(M, N, dtype=AD)
    h = r1.clone()
    ops.linear(x, w, ops.make_ep(h, bias=bias, res1=h, a_res1=0.5, res2=r2, a_res2=0.25))
    ref = x.double() @ w.double().t() + bias.double() + 0.5 * r1.double() + 0.25 * r2.double()
    assert relerr(h, ref) < 2e-5
    scale = EM.gemm_scale(x, w, bias) + 0.5 * r1.double().abs() + 0.25 * r2.double().abs()
    EM.check(h, ref, scale, "gemm", f"linear {tiles} tiles, 2 residuals in place")


def test_linear_geglu_odd_tiles(ops):
    AD = ops.act_dtype()
    M, K, C4 = 64 * 3 + 5, 320, 384
    x = rnd(M, K, dtype=AD)
    w = rnd(2 * C4, K, scale=K ** -0.5, dtype=AD)
    b = rnd(2 * C4)
    idx = torch.arange(2 * C4).view(2, C4 // 16, 16).permute(1, 0, 2).reshape(-1).cuda()   # 16 value / 16 gate blocks
    out = torch.empty(M, C4, device="cuda", dtype=AD)
    ops.linear(x, w[idx].contiguous(), ops.make_ep(out, bias=b[idx].contiguous(), geglu=True))
    ref, scale, approx = geglu_ref(x, w, b)
    assert relerr(out, ref) < EM.tol16(1.5e-3, AD)
    EM.check(out, ref, scale, "gemm", "linear GEGLU odd tiles", approx=approx)


def geglu_ref(x, w, b):
    """value * gelu(gate) in float64, its scale and the polynomial GELU's stated error (tests/test_ops_gpu.py geglu_ref)."""
    C4 = w.shape[0] // 2
    y = x.double() @ w.double().t() + b.double()
    s = EM.gemm_scale(x, w, b)
    v, g = y[:, :C4], y[:, C4:]
    scale = s[:, :C4] * F.gelu(g).abs() + 1.13 * v.abs() * s[:, C4:]
    return v * F.gelu(g), scale, 1.05e-4 * v.abs() * g.abs().clamp_min(4.0)


# The last row tile holds 5 rows and the last column pair one column (N odd): the elements a wrong guard on rows or columns
# would get wrong. Every other activation row is zero, so the rest of the output is bias (+ residuals) alone; the per-element
# bound checks the ragged corner on its own, where a norm over the whole tensor would hide it.
@pytest.mark.parametrize("schedule", ["cooperative", "pingpong", "geglu"])
def test_ragged_last_tile_per_element(ops, schedule):
    AD = ops.act_dtype()
    K = 320
    if schedule == "geglu":
        M, N = 64 * 4 + 5, 512                         # 16-bit output of N / 2 columns; N % 256 == 0 is required
    else:
        M, N = (128 if schedule == "cooperative" else 64) * 3 + 5, 2 * 128 + 43
    tile = 128 if schedule == "cooperative" else 64
    r0 = (M // tile) * tile                            # first row of the ragged last row tile
    x = rnd(M, K, dtype=AD)
    x[:r0] = 0
    w, b = rnd(N, K, scale=K ** -0.5, dtype=AD), rnd(N)
    if schedule == "geglu":
        idx = torch.arange(N).view(2, N // 32, 16).permute(1, 0, 2).reshape(-1).cuda()
        out = torch.empty(M, N // 2, device="cuda", dtype=AD)
        ops.linear(x, w[idx].contiguous(), ops.make_ep(out, bias=b[idx].contiguous(), geglu=True))
        ref, scale, approx = geglu_ref(x, w, b)
        EM.check(out[r0:], ref[r0:], scale[r0:], "gemm", "GEGLU ragged last row tile", approx=approx[r0:])
        EM.check(out[:, -2:], ref[:, -2:], scale[:, -2:], "gemm", "GEGLU last column pair", approx=approx[:, -2:])
        EM.check(out, ref, scale, "gemm", "GEGLU ragged", approx=approx)
        return
    ld = (N + 7) // 8 * 8
    out = torch.empty(M, ld, device="cuda", dtype=AD)[:, :N]
    ref = x.double() @ w.double().t() + b.double()
    scale = EM.gemm_scale(x, w, b)
    if schedule == "pingpong":                         # both residuals: 16-bit output with residuals takes the ping-pong schedule
        r1, r2 = rnd(M, ld)[:, :N], rnd(M, ld, dtype=AD)[:, :N]
        ops.linear(x, w, ops.make_ep(out, bias=b, res1=r1, a_res1=0.5, res2=r2, a_res2=0.25))
        ref = ref + 0.5 * r1.double() + 0.25 * r2.double()
        scale = scale + 0.5 * r1.double().abs() + 0.25 * r2.double().abs()
    else:
        ops.linear(x, w, ops.make_ep(out, bias=b))
    EM.check(out[r0:], ref[r0:], scale[r0:], "gemm", f"{schedule} ragged last row tile")
    EM.check(out[:, N - 1:], ref[:, N - 1:], scale[:, N - 1:], "gemm", f"{schedule} last (single) column")
    EM.check(out, ref, scale, "gemm", f"{schedule} ragged")


@pytest.mark.parametrize("G,M", [(3, 64), (5, 200), (7, 100)])
def test_bmm_nt_odd_batch(ops, G, M):
    AD = ops.act_dtype()
    K, N = 192, 300
    a, b = rnd(G, M, K, dtype=AD), rnd(G, N, K, scale=K ** -0.5, dtype=AD)
    out = torch.empty(G * M, N, device="cuda")
    ops.bmm_nt(a, b, ops.make_ep(out))
    ref = torch.bmm(a.double(), b.double().transpose(1, 2)).reshape(G * M, N)
    assert relerr(out, ref) < 2e-5
    scale = torch.bmm(a.double().abs(), b.double().abs().transpose(1, 2)).reshape(G * M, N)
    EM.check(out, ref, scale, "gemm", f"bmm_nt G={G} M={M}")


@pytest.mark.parametrize("n,H,W", [(3, 3, 64), (5, 1, 64), (2, 9, 16), (3, 22, 32)])
@pytest.mark.parametrize("out_f32", [True, False])
def test_fused_groupnorm_stats_64_row_images(ops, n, H, W, out_f32):
    """Images of an odd number of 64-row tiles: every second image boundary falls inside what a 128-row tile would cover.
    Each consumer warpgroup keeps its own per-image sums and flushes them when its own tile stream changes image."""
    AD = ops.act_dtype()
    C, Co = 64, 320
    x = rnd(n, H, W, C, dtype=AD)
    wp = rnd(Co, 9 * C, scale=(9 * C) ** -0.5, dtype=AD)
    bias = rnd(Co)
    out = torch.empty(n * H * W, Co, device="cuda", dtype=torch.float32 if out_f32 else AD)
    st = torch.zeros(n * 64, device="cuda", dtype=torch.float64)
    produced = ops.conv2d_3x3(x, wp, ops.make_ep(out, bias=bias, gn_stats=(st, Co // 32, 32, H * W)))
    w4 = wp.double().view(Co, 3, 3, C).permute(0, 3, 1, 2)
    ref_out = F.conv2d(x.double().permute(0, 3, 1, 2), w4, bias.double(), padding=1).permute(0, 2, 3, 1).reshape(n * H * W, Co)
    assert relerr(out, ref_out) < (3e-5 if out_f32 else EM.tol16(1e-3, AD))
    scale = F.conv2d(x.double().abs().permute(0, 3, 1, 2), w4.abs(), bias.double().abs(), padding=1)
    EM.check(out, ref_out, scale.permute(0, 2, 3, 1).reshape(n * H * W, Co), "gemm", f"conv3x3 {n}x{H}x{W}")
    if out_f32 and (H * W) % 64 == 0:              # fp32 output: 64-row tiles, one image per tile
        assert produced
    if produced:
        v = out.double().view(n, H * W, 32, Co // 32)
        ref = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1).reshape(-1)
        assert torch.allclose(st, ref, rtol=1e-5, atol=1e-3)


# Fused GroupNorm statistics of outputs whose groups have a mean R times their spread, the offset planted through the bias,
# through res1 or through a per-image row vector (the time-embedding row of the UNet ResBlock's first conv). A 16-bit output
# without a residual runs the cooperative schedule, an fp32 output or one with a residual the ping-pong schedule. Shapes: the
# 64-row images above (ping-pong only: a 128-row tile cannot keep them apart), one image per 128-row tile, and the per-CTA
# accumulation shapes of test_ops_gpu.py::test_fused_groupnorm_stats_accumulated (conv 3x3 and Conv3d (3,1,1)).
def _large_mean_cases():
    cases = []
    for n, H, W, Co, temporal, pp_only, Rs in [(3, 3, 64, 320, False, True, (1e2, 1e3, 1e4)),
                                               (5, 1, 64, 320, False, True, (1e2, 1e3, 1e4)),
                                               (3, 22, 32, 320, False, True, (1e2, 1e3, 1e4)),
                                               (3, 8, 128, 320, False, False, (1e2, 1e3, 1e4)),
                                               (2, 192, 512, 128, False, False, (1e4,)),
                                               (4, 1, 48 * 512, 128, True, False, (1e4,))]:
        for plant in ("bias", "res1", "rowvec"):
            for R in Rs:                                   # float32 output: ping-pong
                cases.append((n, H, W, Co, temporal, plant, R))
            if plant == "res1" or not pp_only:             # 16-bit output: ping-pong with res1, else cooperative
                cases.append((n, H, W, Co, temporal, plant, "16-bit"))
    return cases


@pytest.mark.parametrize("n,H,W,Co,temporal,plant,R", _large_mean_cases())
def test_fused_groupnorm_stats_large_mean(ops, n, H, W, Co, temporal, plant, R):
    AD = ops.act_dtype()
    out_f32 = R != "16-bit"
    R, sigma = (R, 1.0) if out_f32 else large_mean_16(AD)
    C, rpi = 64, H * W
    if temporal:                                   # Conv3d (3,1,1) over [B=1, T=n, H*W, C]; statistics over the whole clip
        x = rnd(1, n, H * W, C, dtype=AD)
        wp = rnd(Co, 3 * C, scale=sigma * (3 * C) ** -0.5, dtype=AD)
        n, rpi = 1, n * H * W
        run = lambda ep: ops.conv_t3(x, wp, ep)
    else:
        x = rnd(n, H, W, C, dtype=AD)
        wp = rnd(Co, 9 * C, scale=sigma * (9 * C) ** -0.5, dtype=AD)
        run = lambda ep: ops.conv2d_3x3(x, wp, ep)
    rows = n * rpi
    offset = offset_tensor(n, Co, R, 0.005 * sigma)  # per image and channel: R + ~1 % of sigma
    bias = offset[0].contiguous() if plant == "bias" else rnd(Co, scale=0.01 * sigma)
    res1 = offset.repeat_interleave(rpi, 0) if plant == "res1" else None
    rowvec = offset if plant == "rowvec" else None
    out = torch.empty(rows, Co, device="cuda", dtype=torch.float32 if out_f32 else AD)
    st = torch.zeros(n * 64, device="cuda", dtype=torch.float64)
    assert run(ops.make_ep(out, bias=bias, rowvec=rowvec, rows_per_vec=rpi, res1=res1, gn_stats=(st, Co // 32, 32, rpi)))
    name = f"fused statistics {'t3' if temporal else 'conv3x3'} {rows}x{Co} {out.dtype} offset in {plant} R={R:g}"
    _, _, ratio = check_group_stats(st, out, n, rpi, Co, name)
    assert ratio.min() > 0.5 * R / sigma, ratio.min()
    g, b = rnd(Co) * 0.1 + 1, rnd(Co) * 0.1
    y = torch.empty(rows, Co, device="cuda", dtype=AD)
    for silu in (False, True):
        ops.groupnorm(out, n, rpi, Co, g, b, 1e-5, silu, y, st, have_stats=True)
        ref, scale = groupnorm_ref(out, n, rpi, Co, g, b, silu)
        EM.check(y, ref, scale, "norm", name + (" SiLU" if silu else ""))
