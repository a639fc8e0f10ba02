"""ctypes binding of libcvvae_b200.so (declarations mirror include/cvvae_b200.h one to one).

There is no CPU fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

from ._build import LIBPATH

F16, BF16, F32 = 0, 1, 2
PAD_ZERO, PAD_REPLICATE = 0, 1
CONV_BIAS_ALONG_M, CONV_FORCE_DIRECT, CONV_OUT_F32, CONV_W_PER_BATCH, CONV_X_SHARED = 1, 2, 4, 8, 16
ABI_VERSION = 3


class Tensor5(C.Structure):
    _fields_ = [
        ("ptr", C.c_void_p),
        ("B", C.c_int32), ("T", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("s_b", C.c_int64), ("s_t", C.c_int64), ("s_h", C.c_int64), ("s_w", C.c_int64), ("s_c", C.c_int64),
    ]


class ConvDesc(C.Structure):
    _fields_ = [
        ("x", Tensor5), ("y", Tensor5),
        ("w", C.c_void_p), ("w_ld", C.c_int64), ("bias", C.c_void_p), ("residual", C.c_void_p),
        ("Cout", C.c_int32),
        ("KT", C.c_int32), ("KH", C.c_int32), ("KW", C.c_int32),
        ("st", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
        ("off_t", C.c_int32), ("off_h", C.c_int32), ("off_w", C.c_int32),
        ("pad_t", C.c_int32), ("pad_hw", C.c_int32),
        ("up_time", C.c_int32), ("dtype", C.c_int32), ("flags", C.c_int32),
        ("alpha", C.c_float),
        ("gn_stats", C.c_void_p), ("gn_groups", C.c_int32),
        ("x2", Tensor5), ("w2", C.c_void_p),
    ]


_P5 = C.POINTER(Tensor5)
_SIGNATURES = {
    "cvvae_conv3d": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "cvvae_conv3d_tc": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "cvvae_conv3d_direct": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "cvvae_conv3d_is_tc": (C.c_int, [C.POINTER(ConvDesc)]),
    "cvvae_conv3d_stacked": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "cvvae_pack_conv_weight": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_groupnorm_stats": (C.c_int, [_P5, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "cvvae_groupnorm_apply": (C.c_int, [_P5, _P5, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                        C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_layernorm": (C.c_int, [_P5, _P5, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_void_p]),
    "cvvae_softmax_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_attn_temporal": (C.c_int, [_P5, _P5, _P5, _P5, C.c_int32, C.c_void_p]),
    "cvvae_replicate_border": (C.c_int, [_P5, C.c_int32, C.c_void_p]),
    "cvvae_copy5": (C.c_int, [_P5, _P5, C.c_int32, C.c_void_p]),
    "cvvae_pack_taps_hw": (C.c_int, [_P5, _P5, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_blend": (C.c_int, [_P5, _P5, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_video_u8_to_f16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_video_f16_to_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_video_resize_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_void_p]),
    "cvvae_video_train_input": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "cvvae_frame_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "cvvae_conv_tc_set_trace": (C.c_int, [C.c_void_p, C.c_int32]),
    "cvvae_conv_tc_plan": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(C.c_int32), C.c_int32]),
    "cvvae_last_error": (C.c_char_p, []),
    "cvvae_abi_version": (C.c_int, []),
    "cvvae_launch_count": (C.c_int64, []),
    "cvvae_probe_umma_shift": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
}
EXPORTS = tuple(_SIGNATURES)
# the values cvvae_conv_tc_plan() writes, in order
CONV_TC_PLAN_FIELDS = ("eligible", "N_cta", "NACC", "TW", "ROWS", "TH", "tiles_w", "tiles_h", "n_tiles_n", "flat", "NA", "NB",
                       "grid", "vec2")
# ... followed by which epilogue the launch runs (1: shared-memory staging and TMA stores)
CONV_TC_PLAN_EPILOGUE_FIELDS = CONV_TC_PLAN_FIELDS + ("tma_epilogue",)

_lib = None


class CvvaeError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the shared library (once). Raises if it has not been built - there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIBPATH):
        raise CvvaeError(
            f"{LIBPATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(cvvae_b200 has no CPU or PyTorch fallback path)")
    lib = C.CDLL(LIBPATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.cvvae_abi_version() != ABI_VERSION:
        raise CvvaeError(f"ABI mismatch: library {lib.cvvae_abi_version()} vs binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().cvvae_last_error().decode(errors="replace")
        raise CvvaeError(f"{what} failed ({rc}): {msg}")
