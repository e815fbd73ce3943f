"""ctypes binding of libtooncrafter_b200.so (the C ABI declared in include/tooncrafter_b200.h).

The product path has no CPU fallback: if the library is missing or a call fails, we raise.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

TC_MAX_TAPS = 9
TC_EPI_GEGLU = 1

_LIB = None


class TcError(RuntimeError):
    pass


class TcConvGemm(C.Structure):
    _fields_ = [
        ("a", C.c_void_p),
        ("a_N", C.c_int), ("a_H", C.c_int), ("a_W", C.c_int), ("a_C", C.c_int),
        ("a_sN", C.c_longlong), ("a_sH", C.c_longlong), ("a_sW", C.c_longlong),
        ("b", C.c_void_p),
        ("b_rows", C.c_int),
        ("ldb", C.c_longlong),
        ("taps", C.c_int),
        ("tap_dx", C.c_int * TC_MAX_TAPS), ("tap_dy", C.c_int * TC_MAX_TAPS), ("tap_dn", C.c_int * TC_MAX_TAPS),
        ("oN", C.c_int), ("oH", C.c_int), ("oW", C.c_int),
        ("out", C.c_void_p),
        ("ldc", C.c_longlong),
        ("n_cols", C.c_int),
        ("bias", C.c_void_p),
        ("bias2", C.c_void_p),
        ("bias2_ld", C.c_longlong),
        ("bias2_rows_per", C.c_int),
        ("res", C.c_void_p),
        ("ldr", C.c_longlong),
        ("acc_scale", C.c_float),
        ("flags", C.c_int),
        ("block_n", C.c_int),
        ("ln_stats", C.c_void_p),
        ("ln_u", C.c_void_p),
        ("ln_nslots", C.c_int),
        ("ln_eps", C.c_float),
        ("row_stats", C.c_void_p),
        ("row_stats_slots", C.c_int),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_longlong),
    ]


class TcAttention(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_longlong), ("q_batches", C.c_int), ("Lq", C.c_int), ("heads", C.c_int),
        ("n_seg", C.c_int),
        ("k", C.c_void_p * 2), ("v", C.c_void_p * 2), ("ldk", C.c_longlong * 2), ("ldv", C.c_longlong * 2),
        ("Lk", C.c_int * 2), ("kv_div", C.c_int * 2),
        ("out", C.c_void_p), ("ldo", C.c_longlong),
        ("scale", C.c_float),
        ("head_dim", C.c_int), ("causal", C.c_int),
    ]


_PROTOTYPES = {
    "tc_last_error": (C.c_char_p, []),
    "tc_version": (C.c_int, []),
    "tc_launch_count": (C.c_ulonglong, []),
    "tc_sm_count": (C.c_int, []),
    "tc_conv_gemm": (C.c_int, [C.POINTER(TcConvGemm), C.c_void_p]),
    "tc_debug_set_gemm_mode": (C.c_int, [C.c_int]),
    "tc_debug_last_gemm_config": (C.c_int, [C.POINTER(C.c_int)]),
    "tc_debug_read_gemm_trace": (C.c_int, [C.c_void_p, C.c_int]),
    "tc_debug_read_attn_trace": (C.c_int, [C.c_void_p, C.c_int]),
    "tc_groupnorm": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p,
                               C.c_void_p]),
    "tc_row_stats": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]),
    "tc_layernorm": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "tc_attention": (C.c_int, [C.POINTER(TcAttention), C.c_void_p]),
    "tc_temporal_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p,
                                        C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "tc_softmax_rows": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "tc_attention_wide": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_longlong, C.c_longlong,
                                    C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "tc_ncthw_to_cl": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.c_int, C.c_float, C.c_void_p]),
    "tc_cl_to_ncthw": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.c_int, C.c_int, C.c_void_p]),
    "tc_upsample2x": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "tc_phase_split2": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "tc_copy2d": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_longlong, C.c_int,
                            C.c_void_p]),
    "tc_add2d": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_longlong, C.c_int,
                           C.c_void_p]),
    "tc_gelu2d": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p]),
    "tc_video_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                              C.c_void_p]),
    "tc_time_embed": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "tc_small_linear": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                  C.c_longlong, C.c_int, C.c_void_p]),
    "tc_ddim_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    "tc_ddim_step3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    "tc_dpm_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    "tc_dpm_step3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]),
    "tc_q_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                              C.c_longlong, C.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_PROTOTYPES.keys())


def lib_path() -> Path:
    import os
    override = os.environ.get("TC_LIB_PATH")          # A/B runs of two builds on one box (scripts/, profiling only)
    if override:
        return Path(override).resolve()
    return Path(__file__).resolve().parent / "libtooncrafter_b200.so"


def load(build_if_missing: bool = True):
    """Load (building first if needed) the CUDA library; raises TcError when unavailable."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if build_if_missing:
        from . import build as _build
        try:
            _build.build()
        except Exception as e:  # nvcc absent on the GPU box is fine when the .so travelled with the snapshot
            if not path.exists():
                raise TcError(f"libtooncrafter_b200.so missing and build failed: {e}") from e
    if not path.exists():
        raise TcError(f"{path} not found: the CUDA extension is required (no CPU fallback)")
    lib = C.CDLL(str(path))
    for name, (res, args) in _PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().tc_last_error()
        raise TcError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
