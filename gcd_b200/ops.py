"""Thin torch-tensor front end over the C ABI (include/gcd_b200.h). Tensors are only used for device memory and the
current CUDA stream; every op launches hand-written sm_90a kernels from libgcd_b200.so. No fallbacks."""
import ctypes

import torch

from . import _lib
from ._lib import Epilogue, TcOp, check


def lib():
    return _lib.load()


_ACT = None


def act_dtype():
    """torch dtype of the 16-bit tensor-core operands the library was built for."""
    global _ACT
    if _ACT is None:
        _ACT = torch.bfloat16 if lib().gcd_act_dtype() == 1 else torch.float16
    return _ACT


# ---- optional per-kernel-class timing (CUDA events on the launching stream); used by bench.py for `roofline` ----
_PROF = None
DETAIL = False   # per-shape names for tc_gemm launches while profiling (tools/prof_forward.py)


class profile:
    """with ops.profile() as prof: ...  -> prof.summary() = {class: {ms, launches, flops, bytes}} (after a sync)."""

    def __enter__(self):
        global _PROF
        self.recs = []
        _PROF = self.recs
        return self

    def __exit__(self, *exc):
        global _PROF
        _PROF = None

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1, fl, by in self.recs:
            d = out.setdefault(name, dict(ms=0.0, launches=0, flops=0.0, bytes=0.0))
            d["ms"] += e0.elapsed_time(e1)
            d["launches"] += 1
            d["flops"] += fl
            d["bytes"] += by
        return out


class _timed:
    __slots__ = ("name", "fl", "by", "e0")

    def __init__(self, name, fl=0.0, by=0.0):
        self.name, self.fl, self.by = name, fl, by

    def __enter__(self):
        if _PROF is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if _PROF is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _PROF.append((self.name, self.e0, e1, self.fl, self.by))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.GcdError("gcd_b200 ops need CUDA tensors (there is no CPU path)")


def _is_f32(t):
    if t.dtype == torch.float32:
        return 1
    if t.dtype == act_dtype():
        return 0
    raise _lib.GcdError(f"unsupported dtype {t.dtype} (expected float32 or {act_dtype()})")


def _ld(t):
    assert t.stride(-1) == 1, "last dim must be contiguous"
    return t.stride(-2) if t.dim() >= 2 else t.numel()


def make_ep(out, bias=None, rowvec=None, rows_per_vec=1, res1=None, a_res1=1.0, res2=None, a_res2=1.0, a_acc=1.0,
            geglu=False, act=0, gn_stats=None):
    """Fused epilogue descriptor; `out`/`res*` are 2-D [rows, cols] views (row stride = leading dimension)."""
    _need_cuda(out, bias, rowvec, res1, res2)
    e = Epilogue()
    e.bias = None if bias is None else bias.data_ptr()
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    e.rowvec = None if rowvec is None else rowvec.data_ptr()
    if rowvec is not None:
        assert rowvec.dtype == torch.float32 and rowvec.dim() == 2 and rowvec.stride(1) == 1
        e.ld_rowvec = rowvec.stride(0)
    e.rows_per_vec = int(rows_per_vec)
    if res1 is not None:
        e.res1, e.ld_res1, e.res1_f32 = res1.data_ptr(), _ld(res1), _is_f32(res1)
    if res2 is not None:
        e.res2, e.ld_res2, e.res2_f32 = res2.data_ptr(), _ld(res2), _is_f32(res2)
    e.a_acc, e.a_res1, e.a_res2 = float(a_acc), float(a_res1), float(a_res2)
    e.out, e.ld_out, e.out_f32 = out.data_ptr(), _ld(out), _is_f32(out)
    e.geglu, e.act = int(bool(geglu)), int(act)
    if gn_stats is not None:      # (float64 buffer [n_img*groups*2] zeroed by the caller, cpg, groups, rows_per_img)
        buf, cpg, groups, rpi = gn_stats
        assert buf.dtype == torch.float64 and buf.is_cuda
        e.gn_stats, e.gn_cpg, e.gn_groups, e.gn_rows_per_img = buf.data_ptr(), int(cpg), int(groups), int(rpi)
    return e


def tc_run(A, C, in_ext, in_strides, out_ext, taps, W, ldw, N, ep, in_mul=1, gemm_tile=False, w_batch_stride=0):
    _need_cuda(A, W)
    assert A.dtype == act_dtype() and W.dtype == act_dtype(), (A.dtype, W.dtype)
    op = TcOp()
    op.A, op.C = A.data_ptr(), int(C)
    op.Xi, op.Yi, op.Zi = [int(v) for v in in_ext]
    op.sx, op.sy, op.sz = [int(v) for v in in_strides]
    op.Xo, op.Yo, op.Zo = [int(v) for v in out_ext]
    op.in_mul, op.ntaps = int(in_mul), len(taps)
    for i, (dx, dy, dz) in enumerate(taps):
        op.tap_dx[i], op.tap_dy[i], op.tap_dz[i] = dx, dy, dz
    op.gemm_tile = int(bool(gemm_tile))
    op.W, op.ldw, op.w_batch_stride, op.N = W.data_ptr(), int(ldw), int(w_batch_stride), int(N)
    op.ep = ep
    name = "tc_gemm"
    if _PROF is not None and DETAIL:
        name = f"tc M{op.Xo * op.Yo * op.Zo} N{op.N} K{op.ntaps * op.C} taps{op.ntaps} g{ep.geglu} r{int(bool(ep.res1))}{int(bool(ep.res2))} o{ep.out_f32}"
    with _timed(name, 2.0 * op.Xo * op.Yo * op.Zo * op.N * op.ntaps * op.C):
        rc = lib().gcd_tc_run(ctypes.byref(op), _stream())
    if rc < 0:
        check(rc, "gcd_tc_run")
    return rc == 0      # False: succeeded, but the requested fused GroupNorm statistics were not produced


def linear(x, w, ep):
    """x: act [rows, K] (row stride arbitrary multiple of 8), w: act [N, K]. nn.Linear / 1x1 conv."""
    rows, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K and w.stride(1) == 1 and x.stride(1) == 1
    sx = x.stride(0)
    return tc_run(x, K, (rows, 1, 1), (sx, sx * rows, sx * rows), (rows, 1, 1), [(0, 0, 0)], w, w.stride(0), N, ep,
                  gemm_tile=True)


def bmm_nt(a, b, ep):
    """a: act [G, M, K], b: act [G, N, K] -> out rows g*M+m, cols n  (torch.bmm(a, b.transpose(1,2)))."""
    G, M, K = a.shape
    N = b.shape[1]
    assert b.shape[0] == G and b.shape[2] == K and a.stride(2) == 1 and b.stride(2) == 1
    tc_run(a, K, (M, G, 1), (a.stride(1), a.stride(0), a.stride(0) * G), (M, G, 1), [(0, 0, 0)], b, b.stride(1), N, ep,
           gemm_tile=True, w_batch_stride=b.stride(0))


TAPS_3x3 = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
TAPS_T3 = [(0, kt - 1, 0) for kt in range(3)]


def conv2d_3x3(x, w, ep, stride=1):
    """x: act [n, H, W, C] channels-last contiguous; w: act [Cout, 9*C] packed (ky, kx, c). padding 1."""
    n, H, W_, C = x.shape
    assert x.is_contiguous() and w.shape[1] == 9 * C
    Ho = (H - 1) // stride + 1
    Wo = (W_ - 1) // stride + 1
    return tc_run(x, C, (W_, H, n), (C, W_ * C, H * W_ * C), (Wo, Ho, n), TAPS_3x3, w, w.stride(0), w.shape[0], ep,
                  in_mul=stride)


TAPS_3x3_PAD01 = [(kx, ky, 0) for ky in range(3) for kx in range(3)]


def conv2d_3x3_down_pad01(x, w, ep):
    """VAE-encoder Downsample (diffusionmodules/model.py:74-91): F.pad(x, (0, 1, 0, 1)) then a 3x3 conv with stride 2 and no
    padding => output (ho, wo) reads input rows 2*ho..2*ho+2, cols 2*wo..2*wo+2; the right/bottom zero column/row is the
    TMA out-of-bounds fill. x: act [n, H, W, C] channels-last; w: act [Cout, 9*C] packed (ky, kx, c)."""
    n, H, W_, C = x.shape
    assert x.is_contiguous() and w.shape[1] == 9 * C
    Ho, Wo = (H - 2) // 2 + 1, (W_ - 2) // 2 + 1
    return tc_run(x, C, (W_, H, n), (C, W_ * C, H * W_ * C), (Wo, Ho, n), TAPS_3x3_PAD01, w, w.stride(0), w.shape[0], ep,
                  in_mul=2)


def conv_t3(x, w, ep):
    """x: act [B, T, HW, C] contiguous; w: act [Cout, 3*C] packed (kt, c). Conv3d kernel (3,1,1), padding (1,0,0)."""
    B, T, HW, C = x.shape
    assert x.is_contiguous() and w.shape[1] == 3 * C
    return tc_run(x, C, (HW, T, B), (C, HW * C, T * HW * C), (HW, T, B), TAPS_T3, w, w.stride(0), w.shape[0], ep)


# ------------------------------------------------------------------------------------------------ norms
def zero_tensor(t):
    """One memset over a whole (contiguous) workspace tensor."""
    nbytes = t.numel() * t.element_size()
    with _timed("elem", 0.0, nbytes):
        check(lib().gcd_memset_async(_p(t), 0, nbytes, _stream()), "memset")


def groupnorm(x, n_img, rows, C, gamma, beta, eps, silu, out, stats, groups=32, have_stats=False):
    """x: [n_img*rows, C] float32 or act -> out act. stats: float64 scratch [n_img*groups*2]; have_stats=True when a
    producing tensor-core op already accumulated them (gcd_epilogue.gn_stats)."""
    _need_cuda(x, gamma, beta, out, stats)
    L = lib()
    st = _stream()
    nbytes = n_img * groups * 2 * 8
    assert stats.dtype == torch.float64 and stats.numel() * 8 >= nbytes
    f32 = _is_f32(x)
    name = "groupnorm"
    if _PROF is not None and DETAIL:
        name = f"groupnorm n{n_img} rows{rows} C{C} f32={int(f32)} fused_stats={int(have_stats)}"
    with _timed(name, 0.0, n_img * rows * C * (((4 if f32 else 2) * (1 if have_stats else 2)) + 2)):
        if not have_stats:
            check(L.gcd_memset_async(_p(stats), 0, nbytes, st), "memset")
            check(L.gcd_groupnorm_stats(_p(x), f32, n_img, rows, C, groups, _p(stats), st), "groupnorm_stats")
        check(L.gcd_groupnorm_apply(_p(x), f32, n_img, rows, C, groups, _p(stats), _p(gamma), _p(beta), float(eps),
                                    int(bool(silu)), _p(out), st), "groupnorm_apply")


def layernorm(x, gamma, beta, out, eps=1e-5, add=None, add_rows_per=1, add_mod=1, sum_out=None):
    _need_cuda(x, gamma, beta, out, add, sum_out)
    rows, C = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and out.dtype == act_dtype()
    with _timed("layernorm", 0.0, rows * C * (6 + (4 if sum_out is not None else 0))):
        check(lib().gcd_layernorm(_p(x), rows, C, _p(gamma), _p(beta), float(eps), _p(add), int(add_rows_per),
                                  int(add_mod), _p(sum_out), _p(out), _stream()), "layernorm")


def layernorm_f32(x, gamma, beta, out, eps=1e-5, add=None, add_rows_per=1, add_mod=1):
    """LayerNorm written as float32 (the ViT's ln_pre, whose output is the residual stream)."""
    _need_cuda(x, gamma, beta, out, add)
    rows, C = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and out.dtype == torch.float32 and out.is_contiguous()
    with _timed("layernorm", 0.0, rows * C * 8):
        check(lib().gcd_layernorm_f32(_p(x), rows, C, _p(gamma), _p(beta), float(eps), _p(add), int(add_rows_per),
                                      int(add_mod), _p(out), _stream()), "layernorm_f32")


def softmax_rows(x, scale, out):
    _need_cuda(x, out)
    rows, cols = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and out.is_contiguous()
    with _timed("elem", 0.0, rows * cols * 10):
        check(lib().gcd_softmax_rows(_p(x), rows, cols, float(scale), _p(out), _stream()), "softmax_rows")


# ------------------------------------------------------------------------------------------------ attention
def attention_spatial(qkv, frames, tokens, heads, out):
    _need_cuda(qkv, out)
    assert qkv.dtype == act_dtype() and qkv.is_contiguous() and out.is_contiguous()
    with _timed("attn_spatial", 4.0 * frames * heads * tokens * tokens * 64, frames * tokens * heads * 64 * 8):
        check(lib().gcd_attention_spatial(_p(qkv), frames, tokens, heads, _p(out), _stream()), "attention_spatial")


def attention_temporal(qkv, clips, T, tokens, heads, out):
    _need_cuda(qkv, out)
    assert qkv.dtype == act_dtype() and qkv.is_contiguous() and out.is_contiguous()
    with _timed("attn_temporal", 4.0 * clips * tokens * heads * T * T * 64, clips * T * tokens * heads * 64 * 8):
        check(lib().gcd_attention_temporal(_p(qkv), clips, T, tokens, heads, _p(out), _stream()), "attention_temporal")


def attention_d80(qkv, n, L, heads, out):
    """qkv: act [n*L, 3*heads*80] (q | k | v) -> out act [n*L, heads*80] (ViT self-attention, head_dim 80)."""
    _need_cuda(qkv, out)
    assert qkv.dtype == act_dtype() and qkv.is_contiguous() and out.is_contiguous()
    assert qkv.shape == (n * L, 3 * heads * 80) and out.shape == (n * L, heads * 80)
    with _timed("attn_d80", 4.0 * n * heads * L * L * 80, n * L * heads * 80 * 8):
        check(lib().gcd_attention_d80(_p(qkv), n, L, heads, _p(out), _stream()), "attention_d80")


def clip_preprocess(x, taps_x, taps_y, mean_std, out, scratch=None):
    """x: float32 NCHW [n, 3, H, W] in [-1, 1] -> out [n*257, 640] patch matrix, act or float32 (include/gcd_b200.h). taps_*: float32
    device tensors of odd length, or None for no antialias blur; scratch: float32 [2*n*3*H*W] when blurring."""
    _need_cuda(x, taps_x, taps_y, mean_std, out, scratch)
    n, c, H, W = x.shape
    assert c == 3 and x.dtype == torch.float32 and x.is_contiguous()
    assert out.shape == (n * 257, 640) and out.is_contiguous()
    ks_x = 0 if taps_x is None else taps_x.numel()
    ks_y = 0 if taps_y is None else taps_y.numel()
    if ks_x:
        assert scratch is not None and scratch.dtype == torch.float32 and scratch.numel() >= 2 * x.numel()
    with _timed("elem", 0.0, x.numel() * (4 + (16 if ks_x else 0)) + out.numel() * 2):
        check(lib().gcd_clip_preprocess(_p(x), n, H, W, _p(taps_x), ks_x, _p(taps_y), ks_y, _p(scratch), _p(mean_std),
                                        _p(out), _is_f32(out), _stream()), "clip_preprocess")


# ------------------------------------------------------------------------------------------------ elementwise
def cast_to_act(x, out):
    _need_cuda(x, out)
    assert x.dtype == torch.float32 and x.is_contiguous() and out.is_contiguous()
    with _timed("elem", 0.0, x.numel() * 6):
        check(lib().gcd_cast_f32_to_act(_p(x), x.numel(), _p(out), _stream()), "cast")


def upsample2x_to_act(x, n, H, W, C, out):
    _need_cuda(x, out)
    with _timed("elem", 0.0, n * H * W * C * (4 + 8)):
        check(lib().gcd_upsample2x_to_act(_p(x), n, H, W, C, _p(out), _stream()), "upsample2x")


def concat_channels(a, b, out, stats=None, n_img=None, groups=32):
    """out[rows, Ca+Cb] = cat(a, b) along channels (float32). With `stats` (zeroed float64 [n_img*groups*2]) the GroupNorm
    statistics of `out` per (image, group) are accumulated in the same pass."""
    _need_cuda(a, b, out, stats)
    rows = a.shape[0]
    assert a.dtype == torch.float32 and b.dtype == torch.float32 and a.is_contiguous() and b.is_contiguous()
    if stats is None:
        with _timed("elem", 0.0, rows * (a.shape[1] + b.shape[1]) * 8):
            check(lib().gcd_concat_channels(_p(a), a.shape[1], _p(b), b.shape[1], rows, _p(out), _stream()), "concat")
        return
    assert stats.dtype == torch.float64 and rows % n_img == 0 and stats.numel() >= n_img * groups * 2
    C = a.shape[1] + b.shape[1]
    if out.dtype == torch.float32:
        with _timed("groupnorm", 0.0, rows * C * 8):
            check(lib().gcd_concat_channels_stats(_p(a), a.shape[1], _p(b), b.shape[1], n_img, rows // n_img, groups, _p(out),
                                                  _p(stats), _stream()), "concat_stats")
    else:                                             # 16-bit concat only (the consumer reads 16-bit operands)
        assert out.dtype == act_dtype() and out.is_contiguous()
        with _timed("groupnorm", 0.0, rows * C * 6):
            check(lib().gcd_concat_channels_stats_act(_p(a), a.shape[1], _p(b), b.shape[1], n_img, rows // n_img, groups, _p(out),
                                                      _p(stats), _stream()), "concat_stats_act")


def silu_act(x, out):
    _need_cuda(x, out)
    with _timed("elem", 0.0, x.numel() * 4):
        check(lib().gcd_silu_act(_p(x), x.numel(), _p(out), _stream()), "silu")


def silu_f32_to_act(x, out):
    _need_cuda(x, out)
    assert x.dtype == torch.float32
    with _timed("elem", 0.0, x.numel() * 6):
        check(lib().gcd_silu_f32_to_act(_p(x), x.numel(), _p(out), _stream()), "silu_f32")


def nchw_to_act_nhwc(x, N, C, HW, Cpad, out):
    _need_cuda(x, out)
    assert x.dtype == torch.float32 and x.is_contiguous()
    with _timed("elem", 0.0, N * HW * (C * 4 + Cpad * 2)):
        check(lib().gcd_nchw_to_act_nhwc(_p(x), N, C, HW, Cpad, _p(out), _stream()), "nchw_to_act_nhwc")


def nhwc_to_nchw(x, ld, N, C, HW, out):
    _need_cuda(x, out)
    assert x.dtype == torch.float32 and out.dtype == torch.float32 and out.is_contiguous()
    with _timed("elem", 0.0, N * HW * C * 8):
        check(lib().gcd_nhwc_to_nchw_f32(_p(x), ld, N, C, HW, _p(out), _stream()), "nhwc_to_nchw")


def vae_time_mix(x, ld, B, T, HW, w, b, out):
    _need_cuda(x, w, b, out)
    with _timed("elem", 0.0, B * T * HW * (ld * 4 + 3 * 4)):
        check(lib().gcd_vae_time_mix(_p(x), ld, B, T, HW, _p(w), _p(b), _p(out), _stream()), "vae_time_mix")


def timestep_embedding(t, dim, out_act=None, out_f32=None, max_period=10000.0):
    _need_cuda(t, out_act, out_f32)
    assert t.dtype == torch.float32 and t.is_contiguous()
    with _timed("elem", 0.0, t.numel() * dim * 2):
        check(lib().gcd_timestep_embedding(_p(t), t.numel(), dim, float(max_period), _p(out_act), _p(out_f32), _stream()),
              "timestep_embedding")


def spherical_embed(x, w, b, out):
    """x: float32 [n, 3]; w: float32 [dim, 13]; b: float32 [dim] -> out float32 [n, dim] (SphericalEmbedder)."""
    _need_cuda(x, w, b, out)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[-1] == 3 and w.is_contiguous() and w.shape[1] == 13
    check(lib().gcd_spherical_embed(_p(x), x.shape[0], _p(w), _p(b), w.shape[0], _p(out), _stream()), "spherical_embed")


def sampler_prep(x, uc_concat, c_concat, BT, H, W, c_in, out):
    _need_cuda(x, uc_concat, c_concat, out)
    with _timed("elem", 0.0, BT * H * W * (3 * 16 + 2 * 128)):
        check(lib().gcd_sampler_prep(_p(x), _p(uc_concat), _p(c_concat), BT, H, W, float(c_in), _p(out), _stream()),
              "sampler_prep")


def sampler_update(x, net_out, ld_net, BT, T, H, W, c_out, c_skip, sigma, dt, scale):
    _need_cuda(x, net_out, scale)
    assert scale.dtype == torch.float32 and scale.numel() == T, "guidance scale must hold one float32 per frame of a clip"
    with _timed("elem", 0.0, BT * H * W * (2 * 16 + 2 * ld_net * 4)):
        check(lib().gcd_sampler_update(_p(x), _p(net_out), ld_net, BT, T, H, W, float(c_out), float(c_skip), float(sigma),
                                       float(dt), _p(scale), _stream()), "sampler_update")


_REPLAYED = 0


def count_replayed_launches(n):
    """Kernel launches executed by replaying a captured CUDA graph (the library's own counter only sees the capture)."""
    global _REPLAYED
    _REPLAYED += int(n)


def launch_count():
    """Kernels of libgcd_b200.so launched so far: direct launches + nodes of replayed CUDA graphs."""
    return int(lib().gcd_launch_count()) + _REPLAYED
