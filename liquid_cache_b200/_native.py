"""ctypes binding of include/lc_gpu.h (liblc_gpu.so).

There is no fallback: if the shared library is missing, or the process has no sm_90a (H100) device,
every entry point raises. Nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LC_GPU_LIB") or os.path.join(_HERE, "lib", "liblc_gpu.so")  # LC_GPU_LIB: debug builds only

LC_OK = 0
LC_ERR_INVALID = -1
LC_ERR_UNSUPPORTED_TYPE = -2
LC_ERR_UNSUPPORTED_EXPR = -3
LC_ERR_CACHE_FULL = -4
LC_ERR_NOT_FOUND = -5
LC_ERR_CUDA = -6
LC_ERR_OOM = -7
LC_ERR_NO_DEVICE = -8

OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_LIKE, OP_NOT_LIKE, OP_CONST_TRUE, OP_CONST_FALSE = range(10)
OP_IN, OP_NOT_IN = 10, 11  # InListExpr (lit_len values in lit_bytes)
IN_LIST_MAX_VALUES, IN_LIST_MAX_BYTES = 256, 16384  # LC_IN_LIST_MAX_VALUES / LC_IN_LIST_MAX_BYTES
HINT_NONE, HINT_PREDICATE, HINT_SUBSTRING_SEARCH = 0, 1, 2
HINT_EXTRACT = {"Year": 3, "Month": 4, "Day": 5, "DayOfWeek": 6}  # CacheExpression::ExtractDate32 { field }
LIT_I64, LIT_U64, LIT_BYTES, LIT_I128, LIT_F64 = 0, 1, 2, 3, 4
SQUEEZE_CLAMP, SQUEEZE_QUANTIZE = 0, 1
# lc_backing_read: int (*)(void* user, uint64_t offset, uint64_t len, uint8_t* dst)
BACKING_READ = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p)
LIQUID_INTEGER, LIQUID_FLOAT, LIQUID_BYTE_VIEW, LIQUID_DECIMAL = 1, 2, 4, 6


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"liblc_gpu error {code}: {msg}")
        self.code = code


class UnsupportedType(NativeError):
    """transcode returned Err(array): the caller keeps the Arrow array."""


class UnsupportedExpr(NativeError):
    """try_eval_predicate returned None: the caller takes its own fallback."""


class CacheFull(NativeError):
    pass


class Predicate(C.Structure):
    _fields_ = [
        ("op", C.c_int32),
        ("lit_kind", C.c_int32),
        ("lit_i64", C.c_int64),
        ("lit_u64", C.c_uint64),
        ("lit_bytes", C.c_char_p),
        ("lit_len", C.c_uint64),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("entries", C.c_uint64),
        ("hbm_bytes_used", C.c_uint64),
        ("hbm_bytes_budget", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("hbm_bytes_reserved", C.c_uint64),
    ]


_lib = None


def exported_symbols_declared_in_header() -> list[str]:
    """Names of every function include/lc_gpu.h declares (used by the CPU-side ABI test)."""
    import re

    hdr = os.path.join(os.path.dirname(_HERE), "include", "lc_gpu.h")
    text = open(hdr).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(lc_[a-z0-9_]+)\s*\(", text)))


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py build` "
            "(there is no Python/CPU implementation of these operators)"
        )
    l = C.CDLL(LIB_PATH)
    vp, u64, i32, u8p = C.c_void_p, C.c_uint64, C.c_int32, C.POINTER(C.c_uint8)
    u64p = C.POINTER(C.c_uint64)
    l.lc_last_error.restype = C.c_char_p
    l.lc_version.restype = C.c_char_p
    l.lc_ctx_create.argtypes = [C.c_int, u64, C.POINTER(vp)]
    l.lc_ctx_destroy.argtypes = [vp]
    l.lc_ctx_destroy.restype = None
    l.lc_ctx_set_stream.argtypes = [vp, vp]
    l.lc_ctx_synchronize.argtypes = [vp]
    l.lc_ctx_stats.argtypes = [vp, C.POINTER(Stats)]
    l.lc_encode.argtypes = [vp, vp, vp, i32, u64, u64p]
    l.lc_cache_retain.argtypes = [vp, u64, u64p]
    l.lc_release.argtypes = [vp, u64]
    l.lc_release.restype = None
    for f in (l.lc_len, l.lc_memory_size):
        f.argtypes = [vp, u64]
        f.restype = u64
    l.lc_data_type.argtypes = [vp, u64]
    l.lc_data_type.restype = i32
    l.lc_entry_image.argtypes = [vp, u64, vp, u64, u64p]
    l.lc_entry_fsst_table.argtypes = [vp, u64, vp, u64, u64p]
    l.lc_arrow_format.argtypes = [vp, u64, C.c_char_p, C.c_size_t]
    l.lc_to_bytes.argtypes = [vp, u64, vp, u64, u64p]
    l.lc_from_bytes.argtypes = [vp, vp, u64, u64p]
    l.lc_from_bytes_scoped.argtypes = [vp, vp, u64, u64, u64p]
    l.lc_ctx_save_symbol_table.argtypes = [vp, u64, vp, u64, u64p]
    l.lc_ctx_load_symbol_table.argtypes = [vp, u64, vp, u64]
    l.lc_squeeze.argtypes = [vp, u64, C.c_int32, C.c_int32, BACKING_READ, vp, vp, u64, u64p, u64p]
    l.lc_squeezed_info.argtypes = [vp, u64, C.POINTER(u64)]
    l.lc_squeezed_component.argtypes = [vp, u64, C.c_int32, vp, vp]
    l.lc_to_arrow.argtypes = [vp, u64, vp, u64, vp, vp]
    l.lc_eval_predicate.argtypes = [vp, u64, C.POINTER(Predicate), vp, u64, vp, vp, u64p, u64p]
    l.lc_mask_bytes.argtypes = [u64]
    l.lc_mask_bytes.restype = u64
    l.lc_eval_predicate_many.argtypes = [vp, vp, u64, C.POINTER(Predicate), vp, vp, vp, vp, vp, vp, vp]
    l.lc_to_arrow_many.argtypes = [vp, vp, u64, vp, vp, vp]
    l.lc_and_then.argtypes = [vp, vp, u64, vp, u64, vp]
    l.lc_cache_insert.argtypes = [vp, u64, vp, vp, i32]
    l.lc_cache_insert_many.argtypes = [vp, vp, u64, vp, vp, i32]
    l.lc_cache_is_cached.argtypes = [vp, u64]
    l.lc_cache_remove.argtypes = [vp, u64]
    l.lc_cache_reset.argtypes = [vp]
    l.lc_cache_handles.argtypes = [vp, vp, u64, vp]
    l.lc_cache_get.argtypes = [vp, u64, vp, u64, vp, vp]
    l.lc_cache_eval_predicate.argtypes = [vp, u64, C.POINTER(Predicate), vp, u64, vp, vp, u64p, u64p]
    l.lc_scan_begin.argtypes = [vp, u64, vp, C.POINTER(vp)]
    l.lc_scan_reset.argtypes = [vp]
    l.lc_ctx_kernel_timing.argtypes = [vp, C.c_int]
    l.lc_ctx_last_kernel_ms.argtypes = [vp]
    l.lc_ctx_last_kernel_ms.restype = C.c_float
    l.lc_ctx_profile_counters.argtypes = [vp, C.c_int, vp]
    l.lc_scan_set_selection.argtypes = [vp, u64, vp, u64]
    l.lc_scan_filter.argtypes = [vp, vp, C.POINTER(Predicate)]
    l.lc_scan_filter_or.argtypes = [vp, u64, vp, C.POINTER(Predicate), vp]
    l.lc_scan_counts.argtypes = [vp, vp, u64p]
    l.lc_scan_selection.argtypes = [vp, u64, vp]
    l.lc_scan_read.argtypes = [vp, vp, vp, vp]
    l.lc_scan_read_device.argtypes = [vp, vp, vp, u64, vp, vp, u64p, u64p, u64p]
    l.lc_scan_selection_layout.argtypes = [vp, u64p, u64p]
    l.lc_scan_store_selections.argtypes = [vp, vp, u64]
    l.lc_scan_load_selections.argtypes = [vp, vp, u64]
    l.lc_scan_read_async.argtypes = [vp, vp, vp, u64, vp, u64, vp]
    l.lc_scan_read_borrowed.argtypes = [vp, vp, C.POINTER(vp), C.POINTER(vp), u64p, u64p]
    l.lc_scan_end.argtypes = [vp]
    l.lc_scan_end.restype = None
    _lib = l
    return l


def check(rc: int) -> None:
    if rc == LC_OK:
        return
    msg = lib().lc_last_error().decode("utf-8", "replace")
    if rc == LC_ERR_UNSUPPORTED_TYPE:
        raise UnsupportedType(rc, msg)
    if rc == LC_ERR_UNSUPPORTED_EXPR:
        raise UnsupportedExpr(rc, msg)
    if rc == LC_ERR_CACHE_FULL:
        raise CacheFull(rc, msg)
    raise NativeError(rc, msg)
