"""ctypes binding of libsvgb200.so (the C ABI declared in include/svgb200.h).

No fallbacks: if the library is missing or a call fails, we raise.  The oracle is never imported here.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

# SVGB200_LIB lets a bring-up script A/B two builds of the same library in one process launch
_LIB_PATH = Path(os.environ.get("SVGB200_LIB") or Path(__file__).resolve().parent / "_lib" / "libsvgb200.so")
_lib = None


class SvgbError(RuntimeError):
    pass


class Plan(C.Structure):
    """mirror of `struct svgb_plan`"""
    _fields_ = [
        ("kind", C.c_int32), ("BH", C.c_int32), ("S", C.c_int32), ("max_items", C.c_int32),
        ("items_stride", C.c_int32),
        ("mask_mode", C.c_int32), ("m0", C.c_int32), ("m1", C.c_int32), ("m2", C.c_int32),
        ("varlen_items", C.c_int32),
        ("counts_off", C.c_int64), ("items_off", C.c_int64), ("chunks_off", C.c_int64),
        ("bytes", C.c_int64),
    ]


_vp, _i, _f, _ll, _sz = C.c_void_p, C.c_int, C.c_float, C.c_longlong, C.c_size_t
_psz = C.POINTER(C.c_size_t)
_pll = C.POINTER(C.c_longlong)  # a {batch, head, row} stride triple
_pplan = C.POINTER(Plan)

# name -> argtypes (restype is int unless noted).  Kept in declaration order of svgb200.h.
_PROTOS = {
    "svgb_version": [],
    "svgb_device_check": [C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)],
    "svgb_attn_plan_varblock_bytes": [_i, _i, _i, _i, _psz],
    "svgb_attn_plan_varblock": [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_varblock_kv_bytes": [_i, _i, _i, _i, _i, _psz],
    "svgb_attn_plan_varblock_kv": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_varblock_gather": [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_band_bytes": [_i, _psz],
    "svgb_attn_plan_band": [_i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_band_t_bytes": [_i, _psz],
    "svgb_attn_plan_band_t": [_i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_local_varlen_bytes": [_i, _i, _i, _psz],
    "svgb_attn_plan_local_varlen": [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_local_varlen_t": [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_block_varlen": [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_block_varlen_t": [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_kvcache_append": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _pll, _pll, _pll, _pll,
                            _vp],
    "svgb_kvcache_append_e4m3": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _pll, _pll, _pll,
                                 _pll, _vp, _vp, _vp],
    "svgb_kvcache_append_e4m3_rows": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _pll, _pll,
                                      _pll, _pll, _vp, _vp, _vp],
    "svgb_attn_plan_kvcache_bytes": [_i, _i, _i, _i, _i, _i, _psz],
    "svgb_attn_plan_kvcache": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_kvcache_split_bytes": [_i, _i, _i, _i, _i, _i, _i, _psz],
    "svgb_attn_plan_kvcache_split": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_kvcache_block_bytes": [_i, _i, _i, _i, _i, _i, _i, _i, _psz],
    "svgb_attn_plan_kvcache_block": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _pplan, _vp],
    "svgb_attn_plan_kvcache_varlen_bytes": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _psz],
    "svgb_attn_plan_kvcache_varlen": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp,
                                      _sz, _pplan, _vp],
    "svgb_kvcache_append_varlen": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _pll, _pll,
                                   _pll, _pll, _vp, _vp, _i, _vp],
    "svgb_attn_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _f,
                      _pplan, _vp, _vp],
    "svgb_attn_fwd_kv": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _ll, _ll, _f, _pplan, _vp,
                         _vp],
    "svgb_attn_fwd_gqa": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _ll, _ll, _f, _pplan,
                          _vp, _vp],
    "svgb_attn_fwd_strided": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _pll, _pll, _pll, _pll, _f, _pplan,
                              _vp, _vp],
    "svgb_attn_fwd_strided_e4m3": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _pll, _pll, _pll,
                                   _pll, _f, _pplan, _vp, _vp],
    "svgb_quantize_e4m3": [_vp, _i, _vp, _vp, _i, _i, _i, _vp],
    "svgb_attn_fwd_kvcache_e4m3_rows": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _pll, _pll,
                                        _pll, _pll, _f, _pplan, _vp, _vp],
    "svgb_attn_fwd_kvcache_split_bytes": [_i, _i, _i, _i, _psz],
    "svgb_attn_fwd_kvcache_split": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _pll,
                                    _pll, _pll, _pll, _f, _pplan, _vp, _vp, _sz, _vp],
    "svgb_quantize_e4m3_rows": [_vp, _i, _vp, _vp, _i, _i, _i, _ll, _ll, _vp],
    "svgb_attn_bwd_bytes": [_i, _i, _psz],
    "svgb_attn_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _ll, _ll, _f, _pplan, _vp, _pplan,
                      _vp, _vp, _sz, _vp],
    "svgb_attn_bwd_kv_bytes": [_i, _i, _i, _psz],
    "svgb_attn_bwd_kv": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _f,
                         _pplan, _vp, _pplan, _vp, _vp, _sz, _vp],
    "svgb_attn_bwd_gqa_bytes": [_i, _i, _i, _i, _psz],
    "svgb_attn_bwd_gqa": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _f,
                          _pplan, _vp, _pplan, _vp, _vp, _sz, _vp],
    "svgb_attn_bwd_strided_bytes": [_i, _i, _i, _i, _i, _psz],
    "svgb_attn_bwd_strided": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, *[_pll] * 8, _f,
                              _pplan, _vp, _pplan, _vp, _vp, _sz, _vp],
    "svgb_density": [_vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "svgb_argsort_labels_bytes": [_i, _i, _i, _psz],
    "svgb_argsort_labels": [_vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp],
    "svgb_permute_gather": [_vp, _vp, _vp, _i, _i, _i, _vp],
    "svgb_permute_scatter": [_vp, _vp, _vp, _i, _i, _i, _vp],
    "svgb_head_placement": [C.POINTER(_vp), C.POINTER(_vp), _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "svgb_kmeans_bytes": [_i, _i, _i, _i, _psz],
    "svgb_row_sqnorm": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "svgb_kmeans_assign": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _sz, _vp],
    "svgb_kmeans_update": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _sz, _vp],
    "svgb_kmeans_run": [_vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _sz, _vp],
    "svgb_kmeans_run_sorted": [_vp, _ll, _vp, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp],
    "svgb_dynamic_map": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp, _vp],
    "svgb_sample_mse_bytes": [_i, _i, _i, _i, _psz],
    "svgb_sample_mse": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _sz, _vp],
    "svgb_rms_norm": [_vp, _vp, _ll, _i, _f, _i, _vp],
    "svgb_layer_norm": [_vp, _vp, _vp, _ll, _i, _i, _vp],
    "svgb_qk_rope": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "svgb_qkv_prep": [_vp, _vp, _vp, _ll, _ll, _vp, _vp, _vp, _ll, _ll, _i, _i, _i, _i, _i, _i,
                      _vp, _vp, _vp, _vp, _f, _i, _vp, _vp, _i, _i, _i, _vp],
    "svgb_row_norm_bwd_bytes": [_ll, _i, _psz],
    "svgb_rms_norm_bwd": [_vp, _vp, _vp, _vp, _vp, _ll, _i, _f, _i, _vp, _sz, _vp],
    "svgb_layer_norm_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _vp, _sz, _vp],
    "svgb_qk_rope_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "svgb_qkv_prep_bwd_bytes": [_i, _i, _i, _i, _i, _psz],
    "svgb_qkv_prep_bwd": [_vp, _vp, _vp, _ll, _ll, _vp, _vp, _ll, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i,
                          _vp, _vp, _f, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _sz, _vp],
    "svgb_layernorm_modulate": [_vp, _i, _vp, _vp, _i, _f, _vp, _vp, _ll, _vp, _i, _ll, _i, _vp],
    "svgb_rmsnorm_hidden": [_vp, _i, _vp, _i, _f, _vp, _i, _ll, _i, _vp],
    "svgb_modulate_shift": [_vp, _i, _vp, _vp, _ll, _vp, _i, _ll, _i, _vp],
    "svgb_gate_residual": [_vp, _i, _vp, _i, _vp, _ll, _vp, _i, _ll, _i, _vp],
    "svgb_selftest_tile": [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _vp],
}


def lib_path() -> Path:
    return _LIB_PATH


def lib():
    """Load (once) and return the library.  Raises SvgbError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise SvgbError(
            f"{_LIB_PATH} not found: build it with `python sparse-videogen_b200/build.py` "
            "(there is no CPU or PyTorch fallback for the svgb200 kernels)")
    l = C.CDLL(os.fspath(_LIB_PATH))
    l.svgb_last_error.restype = C.c_char_p
    l.svgb_last_error.argtypes = []
    for name, args in _PROTOS.items():
        fn = getattr(l, name)  # AttributeError if the .so lacks a declared symbol
        fn.argtypes = args
        fn.restype = C.c_int
    _lib = l
    return l


def check(rc: int, what: str):
    if rc != 0:
        msg = lib().svgb_last_error().decode(errors="replace")
        raise SvgbError(f"{what} failed (rc={rc}): {msg}")
