"""Per-element error bounds of the library's kernels against float64 references, derived from the operand type.

The reference of an op is computed in float64 from the same 16-bit-rounded inputs the kernel reads. Every element of the
kernel's output y must then satisfy

    |y - ref| <= u_out * |ref| + eta_out + kappa * 2^-24 * scale

- u_out: unit roundoff of the stored type: 2^-11 (fp16), 2^-8 (bf16), 0 for a float32 output;
- eta_out: half the subnormal spacing of a 16-bit stored type (2^-25 in fp16), the rounding error below its normal range;
- scale: float64 sum of the absolute values of the terms that make up the element (|A|.|W|^T + |bias| + ... for a GEMM);
- kappa: one constant per op class (KAPPA), the same for the fp16 and the bf16 build: both accumulate in fp32.

tc_gemm's k-loop adds a one-sided term. Each wgmma k16 step adds 16 products to the fp32 accumulator and rounds toward zero,
so every step loses a little of the running sum P_i (the exact sum after step i), always toward zero. Measured on one H100
80GB HBM3 with all-positive operands, the loss is 2.4-3.8 * 2^-24 |P_i| per step on average over the outputs, and about 4.4
at worst. For zero-mean operands P_i random-walks around zero and these losses stay within kappa. For same-sign
operands P_i grows through the k-loop, and the error grows linearly with K: -1.75 (K / 16) 2^-24 sum |a||w| on average when
the running sum grows evenly (1.5e-4 of the result at K = 23040). The bound of a GEMM whose test computes the running sums adds

    GEMM_STEP * 2^-24 * steps,    steps = sum_i |P_i| <= ceil(K / 16) * scale    (gemm_step_sums)

GEMM_STEP = 8 allows four truncations of under one fp32 ulp (2^-23 |P_i|) per k16 step, about twice the measured worst case.
Tests that leave `steps` out hold the kernel to kappa alone; they use zero-mean operands.

Attention packs its softmax weights P to the 16-bit operand type for the P.V MMA. Besides the relative rounding (u_act), a packed
weight below fp16's normal range keeps only an absolute accuracy: half the subnormal spacing of the packed value. The kernels pack
2^15 P, so that weight is ETA_P = 2^-25 / 2^15 = 2^-40 in units of the largest weight of the row (the flash kernels, whose P is
relative to the row maximum) or of 1 (softmax_rows, whose P is normalised). The output moves by at most ETA_P * c * sum_j |v_j|
with c = p_max or 1 (attention_scale). Packed without the offset, keys 17.3+ nats below a dominant one were flushed to zero, and
a row whose dominant key has |v| ~ 0 and whose other keys carry |v| of 1-4 lost most of its output: up to 110 times the bound
at 9216 keys, measured on one H100 80GB HBM3 (tests/test_attention_edges_gpu.py).

A 16-bit fp16 output whose reference rounds past the fp16 maximum must be exactly the infinity of the reference's sign
(IEEE round-to-nearest); within the accumulation error of the overflow threshold either outcome is accepted. bf16 has
fp32's exponent range, so every bf16 output of these tests must be finite.
"""
import torch

U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 0.0}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 0.0}
EPS32 = 2.0 ** -24                    # fp32 unit roundoff
P_OFFSET = 2.0 ** 15                  # attention packs 2^15 P to 16 bits (largest weight 32768)
ETA_P = {t: e / P_OFFSET for t, e in ETA.items()}   # half the subnormal spacing of packed P, in units of P (2^-40 in fp16)
FP16_OVERFLOW = 65520.0               # the smallest magnitude that rounds to inf in fp16 (65504 + half an ulp)

# kappa per op class, in units of 2^-24 * scale (attention: the scale carries P's 16-bit repack, see attention_scale)
KAPPA = {
    "gemm": 32.0,          # tc_gemm: Linear / conv / bmm with the fused epilogue (fp32 accumulation in the tensor cores)
    "attention": 16.0,     # spatial / temporal / d80 flash attention, softmax_rows + P.V (near one-hot rows with
                           # fp16-subnormal outputs reach ~10); the scale carries P's 16-bit pack, subnormal range included
    "norm": 32.0,          # GroupNorm (fp64 sums from each element on) / LayerNorm (two-pass fp32), fp32 normalisation
    "elementwise": 8.0,    # softmax rows, CLIP preprocessing
}
GEMM_STEP = 8.0            # tc_gemm: round-toward-zero loss per wgmma k16 step, in units of 2^-24 * |running sum|


def tol16(tol_fp16, dtype):
    """A relative-L2 bar stated for an fp16 output, scaled to the unit roundoff of `dtype` (unchanged for fp16)."""
    return tol_fp16 * U[dtype] / U[torch.float16]


def gemm_scale(a, w, *terms):
    """|a| @ |w|^T in float64 plus the absolute values of the additive epilogue terms (broadcast to the output)."""
    s = a.double().abs() @ w.double().abs().t()
    for t in terms:
        s = s + t.double().abs()
    return s


def gemm_step_sums(a, w, step=16):
    """sum over the k-steps of tc_gemm's k-loop of |running sum of a . w| in float64, per output element: a [..., M, K],
    w [..., N, K] with columns in the kernel's k order (the packed (tap, channel) order of a convolution's im2col)."""
    a, w = a.double(), w.double().transpose(-1, -2)
    K = a.shape[-1]
    run = torch.zeros(a.shape[:-1] + w.shape[-1:], dtype=torch.float64, device=a.device)
    total = torch.zeros_like(run)
    for k0 in range(0, K, step):
        run += a[..., k0:k0 + step] @ w[..., k0:k0 + step, :]
        total += run.abs()
    return total


def attention_scale(pv_abs, act_dtype, v_abs=None, c=1.0):
    """Scale of an attention output whose value sum is pv_abs = sum_j p_j |v_j|: the fp32 arithmetic, plus P rounded to the
    16-bit operand type for the P.V MMA (u_act * sum_j p_j |v_j|), plus, when v_abs = sum_j |v_j| is given, packed weights in
    the subnormal range (ETA_P * c * sum_j |v_j|, c = p_max for the flash kernels, 1 for softmax_rows); in units of 2^-24."""
    s = pv_abs * (1.0 + U[act_dtype] / EPS32)
    if v_abs is not None:
        s = s + (ETA_P[act_dtype] / EPS32) * c * v_abs
    return s


def check(y, ref, scale, kappa, name="", approx=None, steps=None):
    """Asserts the per-element bound for kernel output `y` against the float64 reference `ref` (same shape); `approx` adds an
    approximation error a kernel states for itself (a polynomial activation), `steps` tc_gemm's k-loop term (gemm_step_sums,
    times GEMM_STEP). Returns the worst ratio of error to bound over the finite elements, and prints it (pytest -s lists it
    per op and build)."""
    kappa = KAPPA[kappa] if isinstance(kappa, str) else kappa
    ref = ref.double().to(y.device)
    scale = scale.double().to(y.device).expand_as(ref)
    yd = y.double()
    e_acc = kappa * EPS32 * scale
    if steps is not None:
        e_acc = e_acc + GEMM_STEP * EPS32 * steps.double().to(y.device)
    if approx is not None:
        e_acc = e_acc + approx.double().to(y.device)
    bound = U[y.dtype] * ref.abs() + ETA[y.dtype] + e_acc
    if y.dtype == torch.float16:
        must_inf = ref.abs() - e_acc >= FP16_OVERFLOW
        may_inf = ref.abs() + e_acc >= FP16_OVERFLOW
    else:
        must_inf = may_inf = torch.zeros_like(ref, dtype=torch.bool)
    fin = torch.isfinite(yd)
    ok_inf = torch.isinf(yd) & may_inf & (torch.sign(yd) == torch.sign(ref))
    err = (yd - ref).abs()
    bad = (~fin & ~ok_inf) | (must_inf & fin) | (fin & (err > bound))
    chk = fin & ~must_inf
    ratio = (err[chk] / bound[chk].clamp_min(1e-300)).max().item() if chk.any() else 0.0
    if bad.any():
        i = bad.flatten().nonzero()[0].item()
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ref.shape))
        raise AssertionError(f"{name}: {int(bad.sum())} of {ref.numel()} elements outside |y - ref| <= u_out |ref| + "
                             f"eta + {kappa:g} 2^-24 scale{' + k-step term' if steps is not None else ''}; first at {idx}: "
                             f"y {yd[idx].item():.9g}, ref {ref[idx].item():.9g}, "
                             f"bound {bound[idx].item():.3g}, {int(must_inf.sum())} elements must overflow to inf; "
                             f"worst error/bound {ratio:.3g}")
    print(f"error/bound {name} [{y.dtype}]: {ratio:.3f}")
    return ratio
