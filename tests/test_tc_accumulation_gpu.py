"""tc_gemm's fp32 accumulation over the reduction lengths the engines launch, against float64 on the same 16-bit inputs.

The wgmma k-loop keeps one fp32 accumulator per output element for the whole reduction (K / 16 MMA steps). With zero-mean
operands its partial sums random-walk around zero and an error made at every step averages out; with same-sign operands the
partial sums grow steadily through the k-loop and an error that leans one way at every step (round toward zero in the tensor
core's adder) grows with the number of steps. Production operands are of the second kind: the convolutions read
SiLU(GroupNorm(.)) (mean about +0.2, bounded below by -0.28), LPIPS's VGG16 reads post-ReLU features, and the VAE's P.V reads
softmax probabilities.

Every shape of PRODUCTION (the longest reductions of each op kind the UNet, the VAE, the CLIP tower and LPIPS launch) runs
under five operand regimes:
    randn      randn activations x randn weights (the control)
    silu       SiLU(randn) activations x randn weights (the UNet's and the VAE's convolution inputs)
    relu       ReLU(randn) activations x randn weights (LPIPS)
    positive   |randn| x |randn|: every partial sum grows, |ref| = sum |a||w| (the worst case for a one-sided step error)
    cancel     positive, with a bias of minus the column median, so most outputs are O(1) while sum |a||w| is large (the
               rows of a convolution whose taps reach into the zero padding sum fewer terms and cancel less)
and each of them with a 16-bit output (cooperative schedule), an fp32 output (ping-pong), an fp32 output updated in place
through res1 (ping-pong: the residual stream) and a 16-bit output with an fp32 residual (ping-pong), under every tile width
gcd_tc_run can pick for the shape's N. The bound is oracle/error_model.py's "gemm" class plus its k-loop term, GEMM_STEP
times the sum over the k16 steps of |running sum| (EM.gemm_step_sums): each step rounds toward zero. Each case also prints
its worst and its mean signed error in units of 2^-24 * (sum |a||w| + |bias| + |residual|): a one-sided step error shows in
the signed mean long before it reaches the worst case.
"""
import contextlib
import math
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from oracle import error_model as EM
from test_ops_gpu import conv3x3_im2col, conv_t3_im2col


@dataclass(frozen=True)
class Shape:
    name: str
    kind: str          # conv3 (3x3, padding 1), t3 (Conv3d (3,1,1)), linear, bmm (bmm_nt)
    C: int             # input channels (conv3 / t3) or K (linear / bmm)
    N: int
    geom: tuple        # conv3: (n, H, W); t3: (B, T, HW); linear: (M,); bmm: (G, M)
    act: int = 0       # the epilogue activation production runs (3: ReLU)
    source: str = ""

    @property
    def K(self):
        return {"conv3": 9, "t3": 3}.get(self.kind, 1) * self.C

    @property
    def rows(self):
        return math.prod(self.geom)


# The longest reductions of each op kind, with where they are launched (UNET_KUBRIC / VAE_DECODER / VAE_ENCODER / VIT_H14 of
# gcd_b200/spec.py and gcd_b200/clip.py, LPIPS CHNS of gcd_b200/lpips.py). The spatial extents are crops of the production
# levels (W kept where it shapes the tiles), a few hundred rows with a ragged last tile.
PRODUCTION = [
    Shape("unet up3 c1 2560->1280", "conv3", 2560, 1280, (2, 9, 16), source="unet.py _vrb c1: output_blocks.0-2 (9x16 level), "
          "cin = 1280 + skip 1280"),
    Shape("unet up2 c1 1920->1280", "conv3", 1920, 1280, (1, 9, 32), source="unet.py _vrb c1: output_blocks.5 (18x32), "
          "1280 + skip 640"),
    Shape("unet up1 c1 1920->640", "conv3", 1920, 640, (1, 5, 64), source="unet.py _vrb c1: output_blocks.6 (36x64), 1280 + 640"),
    Shape("unet 1280->1280", "conv3", 1280, 1280, (1, 9, 32), source="unet.py _vrb c1/c2 at 1280 channels (input_blocks.7-11, "
          "middle_block, output_blocks.0-5 c2), the 'up' convs of output_blocks.2 and .5, the stride-2 'down' of input_blocks.9"),
    Shape("unet up1 c1 1280->640", "conv3", 1280, 640, (1, 5, 64), source="unet.py _vrb c1: output_blocks.7, 640 + skip 640"),
    Shape("unet up1 c1 960->640", "conv3", 960, 640, (1, 5, 64), source="unet.py _vrb c1: output_blocks.8, 640 + skip 320"),
    Shape("unet up0 c1 960->320", "conv3", 960, 320, (1, 3, 128), source="unet.py _vrb c1: output_blocks.9 (72x128), 640 + 320; "
          "N = 320 runs two 160-column tiles"),
    Shape("unet up0 c1 640->320", "conv3", 640, 320, (1, 3, 128), source="unet.py _vrb c1: output_blocks.10-11, 320 + skip 320"),
    Shape("vae 512->512", "conv3", 512, 512, (1, 5, 72), source="vae.py _res2d c1/c2 at 512 channels (decoder mid, up.3, up.2; "
          "encoder down.2-3, mid) and the decoder's up.3 / up.2 upsample convs"),
    Shape("vae up1 c1 512->256", "conv3", 512, 256, (1, 5, 72), source="vae.py _res2d c1: decoder up.1.block.0"),
    Shape("vae up0 c1 256->128", "conv3", 256, 128, (1, 5, 72), source="vae.py _res2d c1: decoder up.0.block.0 (128-column tiles)"),
    Shape("lpips conv4/5 512->512", "conv3", 512, 512, (2, 7, 24), act=3, source="lpips.py _conv: conv4_2, conv4_3, conv5_1-3 "
          "with the ReLU epilogue"),
    Shape("unet time_stack 1280", "t3", 1280, 1280, (1, 14, 21), source="unet.py _vrb time_stack c1/c2 at 1280 channels"),
    Shape("vae time_stack 512", "t3", 512, 512, (1, 14, 23), source="vae.py DecoderEngine._res time_stack c1/c2 at 512 channels"),
    Shape("ff_out / c_proj 5120->1280", "linear", 5120, 1280, (257,), source="unet.py _ff ff.2 / ff_in.2 at C = 1280 (GEGLU "
          "output 4C); clip.py mlp.c_proj (4 x width 1280), 257 rows = one image's tokens"),
    Shape("unet skip 2560->1280", "linear", 2560, 1280, (288,), source="unet.py _vrb skip (1x1 conv) of output_blocks.0-2"),
    Shape("cross-attention to_v 1024->1280", "linear", 1024, 1280, (28,), source="unet.py cross_attn_vectors attn2.v: "
          "context_dim 1024, one row per frame"),
    Shape("vae attention P.V S=9216", "bmm", 9216, 512, (2, 150), source="vae.py _attn P.V: K = S = 72 x 128 latent tokens of "
          "a 576x1024 frame, N = 512 channels"),
]

REGIMES = ("randn", "silu", "relu", "positive", "cancel")
# (label, fp32 output, residual): a residual or an fp32 output selects the ping-pong schedule, a plain 16-bit output the
# cooperative one (gemm.cu gcd_tc_run)
VARIANTS = (("16-bit cooperative", False, False), ("fp32 ping-pong", True, False),
            ("fp32 in-place residual ping-pong", True, True), ("16-bit + fp32 residual ping-pong", False, True))


def tile_widths(N):
    """Every tile width gcd_tc_run picks for N output columns at some row count: 256 when N % 256 == 0 or N >= 384, and then
    160 as well when N % 160 == 0 (the wave-count rule); otherwise 160 when N % 160 == 0, else 128."""
    if N % 256 == 0 or N >= 384:
        return (256, 160) if N % 160 == 0 else (256,)
    return (160,) if N % 160 == 0 else (128,)


@contextlib.contextmanager
def forced_tile_width(ops, bn):
    ops.lib().gcd_tc_override(bn, 0)
    try:
        yield
    finally:
        ops.lib().gcd_tc_override(0, 0)


def operands(shape, regime, AD, seed):
    """The activation and weight operands in the layouts the op reads, rounded to the operand type."""
    a_shape = {"conv3": shape.geom + (shape.C,), "t3": shape.geom + (shape.C,), "linear": shape.geom + (shape.K,),
               "bmm": shape.geom + (shape.K,)}[shape.kind]
    w_shape = (shape.geom[0], shape.N, shape.K) if shape.kind == "bmm" else (shape.N, shape.K)
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(a_shape, generator=g, device="cuda")
    a = {"randn": z, "silu": F.silu(z), "relu": z.clamp_min(0)}.get(regime, z.abs())
    w = torch.randn(w_shape, generator=g, device="cuda") * shape.K ** -0.5
    if regime in ("positive", "cancel"):
        w = w.abs()
    return a.to(AD).contiguous(), w.to(AD).contiguous()


def reference(shape, a, w):
    """float64 sum_k a w, sum_k |a||w| and the k-loop term (EM.gemm_step_sums) per output element, each [rows, N]."""
    if shape.kind == "bmm":
        ad, wd = a.double(), w.double().transpose(1, 2)
        flat = lambda t: t.reshape(-1, shape.N)
        return flat(torch.bmm(ad, wd)), flat(torch.bmm(ad.abs(), wd.abs())), flat(EM.gemm_step_sums(a, w))
    A = {"conv3": conv3x3_im2col, "t3": conv_t3_im2col}.get(shape.kind, lambda t: t.double())(a)
    Wd = w.double().t()
    return A @ Wd, A.abs() @ Wd.abs(), EM.gemm_step_sums(A, w)


def launch(ops, shape, a, w, ep):
    if shape.kind == "conv3":
        return ops.conv2d_3x3(a, w, ep)
    if shape.kind == "t3":
        return ops.conv_t3(a, w, ep)
    if shape.kind == "linear":
        return ops.linear(a, w, ep)
    return ops.bmm_nt(a, w, ep)


def error_units(y, ref, scale):
    """(worst |y - ref|, mean signed y - ref) in units of 2^-24 * scale."""
    e = (y.double() - ref) / (EM.EPS32 * scale)
    return e.abs().max().item(), e.mean().item()


def run_variants(ops, shape, a, w, acc, S, T, bias, bns, tag):
    """Runs the op under every variant and tile width; returns the failures (every case prints its ratios)."""
    AD = ops.act_dtype()
    rows = shape.rows
    g = torch.Generator(device="cuda").manual_seed(rows * shape.N + shape.K)
    r0 = torch.randn(rows, shape.N, generator=g, device="cuda")
    pre = acc + bias.double()
    post = F.relu(pre) if shape.act == 3 else pre
    failures = []
    for label, out_f32, res in VARIANTS:
        ref = post + r0.double() if res else post
        scale = S + bias.double().abs() + (r0.double().abs() if res else 0.0)
        for bn in bns:
            if out_f32:
                out = r0.clone() if res else torch.empty(rows, shape.N, device="cuda")
            else:
                out = torch.empty(rows, shape.N, device="cuda", dtype=AD)
            res1 = (out if out_f32 else r0) if res else None
            with forced_tile_width(ops, bn):
                launch(ops, shape, a, w, ops.make_ep(out, bias=bias, res1=res1, act=shape.act))
            name = f"{tag} {label} BN={bn}"
            worst, mean = error_units(out, ref, scale)
            try:
                ratio = EM.check(out, ref, scale, "gemm", name, steps=T)
            except AssertionError as e:
                failures.append(str(e))
                ratio = float("nan")
            print(f"accumulation {name} [{out.dtype}]: worst {worst:.2f}, mean signed {mean:+.3f} x 2^-24 sum|a||w|; "
                  f"error/bound {ratio:.3f}")
    return failures


@pytest.fixture(scope="module")
def ops():
    from gcd_b200 import ops as o
    o.lib()
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("shape", PRODUCTION, ids=lambda s: s.name.replace(" ", "_"))
def test_production_reduction(ops, shape, regime):
    AD = ops.act_dtype()
    a, w = operands(shape, regime, AD, seed=zlib.crc32(f"{shape.name}/{regime}".encode()))
    acc, S, T = reference(shape, a, w)
    if regime == "cancel":                  # minus the column median: most outputs O(1), sum |a||w| ~ 0.64 sqrt(K)
        bias = -acc.median(0).values.float()
        assert acc.min() > 0 and (acc + bias.double()).abs().median() < 0.05 * S.median()
    else:
        g = torch.Generator(device="cuda").manual_seed(shape.N)
        bias = torch.randn(shape.N, generator=g, device="cuda")
        if regime == "positive":
            bias = bias.abs()
    if regime == "positive":
        assert torch.equal(acc, S)          # every term is >= 0: |ref| is the whole scale
    tag = f"{shape.name} K={shape.K} N={shape.N} {regime}"
    failures = run_variants(ops, shape, a, w, acc, S, T, bias, tile_widths(shape.N), tag)
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [256, 1024, 4096, 9216, 23040])
@pytest.mark.parametrize("pattern", ["uniform", "front-loaded"])
def test_same_sign_error_growth_with_k(ops, K, pattern):
    """All-positive operands at fixed M and N over K: the signed error per k16 step. "uniform": the running sums grow linearly
    through the k-loop; "front-loaded": the first 64 columns of the activations carry ~80 % of sum |a||w|, so every later step
    adds to a running sum close to the final one (the per-step loss relative to the running sum, unaveraged)."""
    AD = ops.act_dtype()
    shape = Shape(f"linear positive {pattern} K={K}", "linear", K, 256, (320,))
    a, w = operands(shape, "positive", AD, seed=K)
    if pattern == "front-loaded":
        a[:, :64] *= K / 16
    acc, S, T = reference(shape, a, w)
    bias = torch.zeros(shape.N, device="cuda")
    failures = []
    for out_f32 in (True, False):
        out = torch.empty(shape.rows, shape.N, device="cuda", dtype=torch.float32 if out_f32 else AD)
        ops.linear(a, w, ops.make_ep(out, bias=bias))
        worst, mean = error_units(out, acc, S)
        _, mean_t = error_units(out, acc, T)
        try:
            ratio = EM.check(out, acc, S, "gemm", shape.name, steps=T)
        except AssertionError as e:
            failures.append(str(e))
            ratio = float("nan")
        print(f"accumulation growth {pattern} K={K} ({K // 16} k16 steps) [{out.dtype}]: worst {worst:.2f}, mean signed "
              f"{mean:+.3f} ({mean / (K // 16):+.4f} per step) x 2^-24 sum|a||w|, mean signed {mean_t:+.3f} x 2^-24 "
              f"sum_i |P_i|; error/bound {ratio:.3f}")
    assert not failures, "\n".join(failures)


def test_gemm_step_sums_matches_the_k_loop():
    """EM.gemm_step_sums against the running sums written out step by step, for a batched and a plain operand pair."""
    g = torch.Generator().manual_seed(3)
    a, w = torch.randn(2, 5, 40, generator=g), torch.randn(2, 3, 40, generator=g)
    want = torch.zeros(2, 5, 3, dtype=torch.float64)
    for b in range(2):
        for m in range(5):
            for n in range(3):
                p = (a[b, m].double() * w[b, n].double()).tolist()
                run = 0.0
                for k0 in range(0, 40, 16):
                    run += sum(p[k0:k0 + 16])
                    want[b, m, n] += abs(run)
    assert torch.allclose(EM.gemm_step_sums(a, w), want, rtol=1e-12, atol=0)
    assert torch.allclose(EM.gemm_step_sums(a[0], w[0]), want[0], rtol=1e-12, atol=0)


def _engine_shapes():
    """(kind, K, N) of the tensor-core convolutions and the long linears the engines build, from their plans."""
    from gcd_b200 import clip, lpips, spec
    out = set()
    u = spec.UNET_KUBRIC
    inp, mid, outb = spec.unet_plan(u)
    for kind, _, cin, cout in [layer for blk in inp + [mid] + outb for layer in blk]:
        if kind == "vrb":
            out |= {("conv3", 9 * cin, cout), ("conv3", 9 * cout, cout), ("t3", 3 * cout, cout)}
            if cin != cout:
                out.add(("linear", cin, cout))
        elif kind in ("up", "down"):
            out.add(("conv3", 9 * cin, cout))
        elif kind == "svt":
            out |= {("linear", 4 * cout, cout), ("linear", u["context_dim"], cout)}
    for plan in (spec.decoder_plan(spec.VAE_DECODER), spec.encoder_plan(spec.VAE_ENCODER)):
        for kind, _, cin, cout in plan:
            if kind == "res":
                out |= {("conv3", 9 * cin, cout), ("conv3", 9 * cout, cout), ("t3", 3 * cout, cout)}
            elif kind in ("up", "down"):
                out.add(("conv3", 9 * cin, cout))
    cin = 64
    for cout, idx in zip(lpips.CHNS, lpips.SLICES):
        for i in idx:
            if i:
                out.add(("conv3", 9 * cin, cout))
            cin = cout
    out.add(("linear", 4 * clip.VIT_H14["width"], clip.VIT_H14["width"]))
    return out


def test_production_table_matches_the_engine_plans():
    """Every conv / linear row of PRODUCTION is a shape the engines launch, and the table holds the longest reduction of each
    op kind (the VAE's P.V, whose K is the latent token count, is checked against the 576x1024 frame size)."""
    shapes = _engine_shapes()
    table = {(s.kind, s.K, s.N) for s in PRODUCTION}
    assert {t for t in table if t[0] != "bmm"} <= shapes, sorted({t for t in table if t[0] != "bmm"} - shapes)
    for kind in ("conv3", "t3", "linear"):
        longest = max(k for t, k, _ in shapes if t == kind)
        assert any(t == kind and k == longest for t, k, _ in table), (kind, longest)
    from gcd_b200 import spec
    vae = spec.VAE_DECODER
    assert ("bmm", (576 // 8) * (1024 // 8), vae["ch"] * vae["ch_mult"][-1]) in table
