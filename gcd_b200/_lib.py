"""ctypes binding of libgcd_b200.so (the C ABI declared in include/gcd_b200.h).

The CUDA library is the product path: there is NO CPU or eager-PyTorch fallback. Importing this module without the
built library raises; calling any op without a CUDA device raises.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int8, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GCD_LIB_PATH") or os.path.join(_HERE, "libgcd_b200.so")   # override: experiments with variant builds


class GcdError(RuntimeError):
    pass


class Epilogue(Structure):
    _fields_ = [
        ("bias", c_void_p), ("rowvec", c_void_p), ("rows_per_vec", c_int32), ("ld_rowvec", c_int32),
        ("res1", c_void_p), ("ld_res1", c_int32), ("res1_f32", c_int32),
        ("res2", c_void_p), ("ld_res2", c_int32), ("res2_f32", c_int32),
        ("a_acc", c_float), ("a_res1", c_float), ("a_res2", c_float),
        ("out", c_void_p), ("ld_out", c_int32), ("out_f32", c_int32), ("geglu", c_int32), ("act", c_int32),
        ("gn_stats", c_void_p), ("gn_cpg", c_int32), ("gn_groups", c_int32), ("gn_rows_per_img", c_int64),
    ]


class TcOp(Structure):
    _fields_ = [
        ("A", c_void_p), ("C", c_int32), ("Xi", c_int32), ("Yi", c_int32), ("Zi", c_int32),
        ("sx", c_int64), ("sy", c_int64), ("sz", c_int64),
        ("Xo", c_int32), ("Yo", c_int32), ("Zo", c_int32), ("in_mul", c_int32), ("ntaps", c_int32),
        ("tap_dx", c_int8 * 9), ("tap_dy", c_int8 * 9), ("tap_dz", c_int8 * 9),
        ("gemm_tile", c_int32), ("W", c_void_p), ("ldw", c_int64), ("w_batch_stride", c_int64), ("N", c_int32),
        ("ep", Epilogue),
    ]


_SIGS = {
    "gcd_last_error": (c_char_p, []),
    "gcd_version": (c_int, []),
    "gcd_act_dtype": (c_int, []),
    "gcd_launch_count": (c_int64, []),
    "gcd_tc_run": (c_int, [POINTER(TcOp), c_void_p]),
    "gcd_tc_override": (None, [c_int, c_int]),
    "gcd_groupnorm_stats": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "gcd_groupnorm_apply": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_float, c_int, c_void_p, c_void_p]),
    "gcd_layernorm": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int64, c_int64,
                              c_void_p, c_void_p, c_void_p]),
    "gcd_layernorm_f32": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int64, c_int64,
                                  c_void_p, c_void_p]),
    "gcd_attention_spatial": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_attention_d80": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_clip_preprocess": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                    c_void_p, c_int, c_void_p]),
    "gcd_attention_temporal": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_softmax_rows": (c_int, [c_void_p, c_int64, c_int, c_float, c_void_p, c_void_p]),
    "gcd_memset_async": (c_int, [c_void_p, c_int, c_int64, c_void_p]),
    "gcd_cast_f32_to_act": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "gcd_upsample2x_to_act": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_concat_channels": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "gcd_concat_channels_stats": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "gcd_concat_channels_stats_act": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "gcd_silu_act": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "gcd_silu_f32_to_act": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "gcd_nchw_to_act_nhwc": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_nhwc_to_nchw_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_vae_time_mix": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gcd_timestep_embedding": (c_int, [c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "gcd_spherical_embed": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "gcd_frame_metrics": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_render_views": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                 c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gcd_frames_prepare": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p]),
    "gcd_unproject_depth": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p]),
    "gcd_lpips_input": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gcd_maxpool2x2": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gcd_lpips_head": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "gcd_sampler_prep": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "gcd_sampler_update": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_float,
                                   c_float, c_void_p, c_void_p]),
}

EXPORTS = tuple(_SIGS.keys())
MISSING = []      # declared symbols the loaded library does not export (a GCD_LIB_PATH build of older sources)

_lib = None


def load():
    """Loads the shared library (once). Raises GcdError if it has not been built (python -m gcd_b200.build).

    A declared symbol the library does not export is left unbound and listed in MISSING: calling it raises AttributeError
    (undefined symbol), while everything the library does export works. That keeps a variant build of older sources usable
    through GCD_LIB_PATH for the paths it covers (A/B of the sampler against an earlier library); the in-tree build exports
    every symbol (checked by build() and tests/test_host_cpu.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GcdError(f"{LIB_PATH} is missing: build it with `python -m gcd_b200.build` "
                       "(gcd_b200 has no CPU / eager fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    MISSING.clear()
    for name, (res, args) in _SIGS.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            MISSING.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().gcd_last_error()
        raise GcdError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")
