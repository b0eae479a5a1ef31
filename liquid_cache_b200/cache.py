"""Host-side mirror of the reference's cache front door, over the C ABI.

Reference: `LiquidCacheBuilder` (/root/reference/src/core/src/cache/builders.rs:32-158),
`LiquidCache::{insert,get,eval_predicate}` (src/core/src/cache/core.rs:122-142) and the
`Insert` / `Get` / `EvaluatePredicate` builders (builders.rs:162-356). Same names, same argument
meaning, same return conventions (`None` = entry absent; `CacheFull` raised where the reference
returns `Err(CacheFull)`). The reference's builders are `IntoFuture`; here `.read()` / `.run()` play
the part of `.await`.

Everything array-sized happens in liblc_gpu.so on the GPU. This module only moves Arrow arrays across
the Arrow C Data Interface and keeps the EntryID bookkeeping.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import pyarrow as pa
from pyarrow.cffi import ffi as _ffi

from . import _native as N
from .expr import CacheExpression, LiquidExpr


class EntryID(int):
    """`EntryID(usize)` (src/core/src/cache/utils.rs:73-88)."""

    def __new__(cls, v: int):
        return super().__new__(cls, int(v))


def parquet_array_id(file_id: int, rg_id: int, col_id: int, batch_id: int) -> EntryID:
    """`ParquetArrayID` packing: file<<48 | rg<<32 | col<<16 | batch (src/datafusion/src/cache/id.rs:15-22)."""
    return EntryID((file_id << 48) | (rg_id << 32) | (col_id << 16) | batch_id)


# ---- Arrow C Data Interface plumbing ----
def _export(arr: pa.Array):
    c_arr = _ffi.new("struct ArrowArray*")
    c_sch = _ffi.new("struct ArrowSchema*")
    arr._export_to_c(int(_ffi.cast("uintptr_t", c_arr)), int(_ffi.cast("uintptr_t", c_sch)))
    return c_arr, c_sch


def _ptr(cdata) -> int:
    return int(_ffi.cast("uintptr_t", cdata))


def _new_out():
    return _ffi.new("struct ArrowArray*"), _ffi.new("struct ArrowSchema*")


def _import(c_arr, c_sch) -> pa.Array:
    return pa.Array._import_from_c(_ptr(c_arr), _ptr(c_sch))


def selection_bits(sel) -> tuple[Optional[np.ndarray], int]:
    """BooleanBuffer -> (LSB-first bytes at bit offset 0, length). Accepts a pyarrow BooleanArray
    (must have no nulls: a BooleanBuffer cannot), a numpy bool array, or a list of bools."""
    if sel is None:
        return None, 0
    if isinstance(sel, pa.ChunkedArray):
        sel = sel.combine_chunks()
    if isinstance(sel, pa.Array):
        if sel.null_count:
            raise ValueError("a selection is a BooleanBuffer: it cannot have nulls")
        mask = np.asarray(sel.to_numpy(zero_copy_only=False), dtype=bool)
    else:
        mask = np.asarray(sel, dtype=bool)
    n = int(mask.shape[0])
    bits = np.packbits(mask, bitorder="little")
    pad = (-len(bits)) % 8
    if pad or len(bits) == 0:
        bits = np.concatenate([bits, np.zeros(pad or 8, dtype=np.uint8)])
    return np.ascontiguousarray(bits), n


def _mask_to_boolean_array(values: np.ndarray, validity: Optional[np.ndarray], n: int, null_count: int) -> pa.Array:
    vals = np.unpackbits(values, bitorder="little")[:n].astype(bool)
    if null_count == 0 or validity is None:
        return pa.array(vals, type=pa.bool_())
    valid = np.unpackbits(validity, bitorder="little")[:n].astype(bool)
    return pa.array(vals, type=pa.bool_(), mask=~valid)


class GpuLiquidArray:
    """`Arc<dyn LiquidArray>` whose payload lives in HBM (trait LiquidArray,
    src/core/src/liquid_array/mod.rs:82-146)."""

    def __init__(self, cache: "LiquidCache", handle: int, owned: bool = True):
        self._cache = cache
        self._h = handle
        self._owned = owned

    def __del__(self):
        try:
            if self._owned and self._h and self._cache._ctx:
                N.lib().lc_release(self._cache._ctx, self._h)
        except Exception:
            pass

    @property
    def handle(self) -> int:
        return self._h

    def len(self) -> int:
        return int(N.lib().lc_len(self._cache._ctx, self._h))

    __len__ = len

    def get_array_memory_size(self) -> int:
        return int(N.lib().lc_memory_size(self._cache._ctx, self._h))

    def data_type(self) -> int:
        return int(N.lib().lc_data_type(self._cache._ctx, self._h))

    def entry_image(self) -> bytes:
        """The entry's HBM image (csrc/entry_layout.h), copied to the host."""
        nb = C.c_uint64(0)
        N.check(N.lib().lc_entry_image(self._cache._ctx, self._h, None, 0, C.byref(nb)))
        buf = np.zeros(nb.value, dtype=np.uint8)
        N.check(N.lib().lc_entry_image(self._cache._ctx, self._h, buf.ctypes.data, nb.value, C.byref(nb)))
        return buf.tobytes()

    def to_bytes(self) -> bytes:
        """`LiquidArray::to_bytes`: the reference's LQDA image of the entry (Integer / Float / Decimal)."""
        nb = C.c_uint64(0)
        N.check(N.lib().lc_to_bytes(self._cache._ctx, self._h, None, 0, C.byref(nb)))
        buf = np.zeros(max(int(nb.value), 1), dtype=np.uint8)
        N.check(N.lib().lc_to_bytes(self._cache._ctx, self._h, buf.ctypes.data, nb.value, C.byref(nb)))
        return buf[: int(nb.value)].tobytes()

    def squeeze(self, io, expression_hint, policy: str = "clamp"):
        """`LiquidArray::squeeze(io, expression_hint)` (liquid_array/primitive_array.rs:389-499) under
        `IntegerSqueezePolicy::{Clamp, Quantize}`: returns `(squeezed array, full LQDA bytes)` or None when the
        reference would not squeeze. `io` mirrors `SqueezeIoHandler`: `io.read((start, end)) -> bytes` is called when the
        half-width codes cannot answer; the caller stores the returned bytes where `io` will find them."""
        pol = {"clamp": N.SQUEEZE_CLAMP, "quantize": N.SQUEEZE_QUANTIZE}[policy]
        field = CacheExpression.as_date32_field(expression_hint)
        hint = N.HINT_NONE if expression_hint is None else N.HINT_EXTRACT[field] if field else (
            N.HINT_SUBSTRING_SEARCH if expression_hint == CacheExpression.SubstringSearch else N.HINT_PREDICATE)
        nb, sq = C.c_uint64(0), C.c_uint64(0)
        ctx = self._cache._ctx
        N.check(N.lib().lc_squeeze(ctx, self._h, pol, hint, N.BACKING_READ(), None, None, 0, C.byref(nb), C.byref(sq)))  # size query: no reader yet
        if nb.value == 0:
            return None

        def _read(_user, offset, length, dst):
            try:
                data = io.read((int(offset), int(offset + length)))
                if len(data) != length:
                    return 2
                C.memmove(dst, data, length)
                return 0
            except Exception:  # the C side reports the failed read
                return 1

        cb = N.BACKING_READ(_read)
        buf = np.zeros(int(nb.value), dtype=np.uint8)
        N.check(N.lib().lc_squeeze(ctx, self._h, pol, hint, cb, None, buf.ctypes.data, nb.value, C.byref(nb), C.byref(sq)))
        squeezed = GpuSqueezedArray(self._cache, int(sq.value))
        squeezed._keepalive = (cb, io)  # the C side calls back for as long as the entry lives
        return squeezed, buf[: int(nb.value)].tobytes()

    def fsst_table(self) -> bytes:
        """The column chunk's FSST symbol table as the kernels see it (lc::FsstTable: 256 x u64 symbols, 256 x u8 lengths)."""
        nb = C.c_uint64(0)
        N.check(N.lib().lc_entry_fsst_table(self._cache._ctx, self._h, None, 0, C.byref(nb)))
        buf = np.zeros(nb.value, dtype=np.uint8)
        N.check(N.lib().lc_entry_fsst_table(self._cache._ctx, self._h, buf.ctypes.data, nb.value, C.byref(nb)))
        return buf.tobytes()

    def original_arrow_data_type(self) -> pa.DataType:
        return self.to_arrow_array().type if self.len() == 0 else self._type_from_format()

    def _type_from_format(self) -> pa.DataType:
        buf = C.create_string_buffer(64)
        N.check(N.lib().lc_arrow_format(self._cache._ctx, self._h, buf, 64))
        return _type_of_format(buf.value.decode())

    def to_arrow_array(self) -> pa.Array:
        return self.filter(None)

    def filter(self, selection) -> pa.Array:
        bits, n = selection_bits(selection)
        out_a, out_s = _new_out()
        N.check(
            N.lib().lc_to_arrow(
                self._cache._ctx, self._h, bits.ctypes.data if bits is not None else None, n, _ptr(out_s), _ptr(out_a)
            )
        )
        return _import(out_a, out_s)

    def try_eval_predicate(self, expr: LiquidExpr, selection) -> pa.Array:
        pred = expr.to_native(self._type_from_format())
        bits, n = selection_bits(selection)
        rows = self.len()
        nb = int(N.lib().lc_mask_bytes(rows))
        vals = np.zeros(nb, dtype=np.uint8)
        valid = np.zeros(nb, dtype=np.uint8)
        out_len, out_nulls = C.c_uint64(0), C.c_uint64(0)
        N.check(
            N.lib().lc_eval_predicate(
                self._cache._ctx,
                self._h,
                C.byref(pred),
                bits.ctypes.data if bits is not None else None,
                n,
                vals.ctypes.data,
                valid.ctypes.data,
                C.byref(out_len),
                C.byref(out_nulls),
            )
        )
        return _mask_to_boolean_array(vals, valid, int(out_len.value), int(out_nulls.value))


class GpuSqueezedArray(GpuLiquidArray):
    """`LiquidSqueezedArray` (liquid_array/mod.rs:209-263) for the two integer forms: `to_arrow_array`, `filter` and
    `try_eval_predicate` keep their meaning, reading the backing bytes through `io` when the codes cannot answer."""

    def _info(self):
        out = (C.c_uint64 * 6)()
        N.check(N.lib().lc_squeezed_info(self._cache._ctx, self._h, out))
        return [int(x) for x in out]

    def policy(self) -> str:
        return {1: "clamp", 2: "quantize", 3: "date32"}[self._info()[0]]

    def field(self) -> str:
        """`SqueezedDate32Array::field` (squeezed_date32_array.rs:270-272)"""
        assert self._info()[0] == 3
        return ("Year", "Month", "Day", "DayOfWeek")[self._info()[2]]

    def _component(self, lossy: int) -> pa.Array:
        out_a, out_s = _new_out()
        N.check(N.lib().lc_squeezed_component(self._cache._ctx, self._h, lossy, _ptr(out_s), _ptr(out_a)))
        return _import(out_a, out_s)

    def to_component_array(self) -> pa.Array:
        """`SqueezedDate32Array::to_component_array` (:276-282): the column's own type, dates whose component is the
        stored one — no backing read."""
        return self._component(1)

    def to_component_date32(self) -> pa.Array:
        """`to_component_date32` (:286-294): the component values themselves, typed Date32."""
        return self._component(0)

    def bit_width(self) -> int:
        return self._info()[1]

    def bucket_width(self) -> int:
        return self._info()[2]

    def disk_backing(self) -> int:
        """`SqueezedBacking::Liquid(len)`: bytes of the image behind `io`."""
        return self._info()[3]

    def to_bytes(self) -> bytes:
        raise N.UnsupportedType(N.LC_ERR_UNSUPPORTED_TYPE, "a squeezed array has no serialized form; its full image is the backing")


_FORMAT_TO_TYPE = {
    "c": pa.int8(), "s": pa.int16(), "i": pa.int32(), "l": pa.int64(),
    "C": pa.uint8(), "S": pa.uint16(), "I": pa.uint32(), "L": pa.uint64(),
    "tdD": pa.date32(), "tdm": pa.date64(),
    "tss:": pa.timestamp("s"), "tsm:": pa.timestamp("ms"), "tsu:": pa.timestamp("us"), "tsn:": pa.timestamp("ns"),
    "u": pa.string(), "z": pa.binary(), "vu": pa.string_view(), "vz": pa.binary_view(),
    "S:u": pa.dictionary(pa.uint16(), pa.string()), "S:z": pa.dictionary(pa.uint16(), pa.binary()),
}


_FORMAT_TO_TYPE.update({"f": pa.float32(), "g": pa.float64()})


def _type_of_format(fmt: str) -> pa.DataType:
    """Arrow C format string -> pyarrow type; decimals carry their parameters ("d:precision,scale[,bits]")."""
    if fmt.startswith("d:"):
        parts = [int(x) for x in fmt[2:].split(",")]
        bits = parts[2] if len(parts) > 2 else 128
        return pa.decimal256(parts[0], parts[1]) if bits == 256 else pa.decimal128(parts[0], parts[1])
    return _FORMAT_TO_TYPE[fmt]


class LiquidCacheBuilder:
    """`LiquidCacheBuilder` (builders.rs:32-158). Options that configure the reference's CPU-side
    policies (cache/hydration/squeeze policies, disk store) are accepted and recorded but have no
    effect here: an HBM-resident cache never squeezes to disk."""

    def __init__(self):
        self._batch_size = 8192
        self._max_memory_bytes = 0
        self._device = 0
        self._ignored = {}

    @staticmethod
    def new() -> "LiquidCacheBuilder":
        return LiquidCacheBuilder()

    def with_batch_size(self, n: int):
        self._batch_size = int(n)
        return self

    def with_max_memory_bytes(self, n: int):
        self._max_memory_bytes = int(n)
        return self

    def with_device(self, device: int):
        self._device = int(device)
        return self

    def _ignore(name):  # noqa: N805
        def f(self, *a, **k):
            self._ignored[name] = (a, k)
            return self

        return f

    with_max_disk_bytes = _ignore("max_disk_bytes")
    with_cache_policy = _ignore("cache_policy")
    with_hydration_policy = _ignore("hydration_policy")
    with_squeeze_policy = _ignore("squeeze_policy")
    with_metadata = _ignore("metadata")
    with_store = _ignore("store")
    with_squeeze_victims_concurrently = _ignore("squeeze_victims_concurrently")

    def build(self) -> "LiquidCache":
        return LiquidCache(self._device, self._max_memory_bytes, self._batch_size)


class Insert:
    """`Insert` builder (builders.rs:162-214)."""

    def __init__(self, cache, entry_id, array):
        self._cache, self._id, self._array = cache, entry_id, array
        self._hint = None

    def with_skip_gc(self):
        return self

    def with_squeeze_hint(self, hint):
        self._hint = hint
        return self

    def run(self) -> None:
        hint = N.HINT_SUBSTRING_SEARCH if self._hint == CacheExpression.SubstringSearch else (
            N.HINT_PREDICATE if self._hint else N.HINT_NONE)
        c_arr, c_sch = _export(self._array)
        N.check(N.lib().lc_cache_insert(self._cache._ctx, int(self._id), _ptr(c_sch), _ptr(c_arr), hint))
        self._cache._types[int(self._id)] = self._array.type


class Get:
    """`Get` builder (builders.rs:218-276)."""

    def __init__(self, cache, entry_id):
        self._cache, self._id = cache, entry_id
        self._sel = None

    def with_selection(self, selection):
        self._sel = selection
        return self

    def with_expression_hint(self, _hint):
        return self

    def with_optional_expression_hint(self, _hint):
        return self

    def read(self) -> Optional[pa.Array]:
        if not self._cache.is_cached(self._id):
            return None
        bits, n = selection_bits(self._sel)
        out_a, out_s = _new_out()
        N.check(
            N.lib().lc_cache_get(
                self._cache._ctx, int(self._id), bits.ctypes.data if bits is not None else None, n, _ptr(out_s), _ptr(out_a)
            )
        )
        return _import(out_a, out_s)


class EvaluatePredicate:
    """`EvaluatePredicate` builder (builders.rs:314-356)."""

    def __init__(self, cache, entry_id, expr: LiquidExpr):
        self._cache, self._id, self._expr = cache, entry_id, expr
        self._sel = None

    def with_selection(self, selection):
        self._sel = selection
        return self

    def read(self) -> Optional[pa.Array]:
        if not self._cache.is_cached(self._id):
            return None
        arr = self._cache.try_read_liquid(self._id)  # holds its own reference for the duration of the call
        if arr is None:
            return None
        return arr.try_eval_predicate(self._expr, self._sel)


class LiquidCache:
    """`LiquidCache` (core.rs:52-277) with its entries resident in the HBM of ONE device."""

    def __init__(self, device: int = 0, max_memory_bytes: int = 0, batch_size: int = 8192):
        self._ctx = None
        ctx = C.c_void_p()
        N.check(N.lib().lc_ctx_create(device, max_memory_bytes, C.byref(ctx)))
        self._ctx = ctx
        self._batch_size = batch_size
        self._types: dict[int, pa.DataType] = {}

    def close(self):
        if self._ctx:
            N.lib().lc_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def batch_size(self) -> int:
        return self._batch_size

    # -- reference front door --
    def insert(self, entry_id, array: pa.Array) -> Insert:
        return Insert(self, entry_id, array)

    def insert_many(self, entry_ids: Sequence[int], arrays: Sequence[pa.Array], hint=None) -> None:
        """`insert` for a list of batches in one call (lc_cache_insert_many): integer-like batches are transcoded in
        one pass on the device. All or nothing."""
        n = len(entry_ids)
        if n != len(arrays):
            raise ValueError("entry_ids and arrays differ in length")
        if n == 0:
            return
        exported = [_export(a) for a in arrays]  # keeps the C structs alive for the duration of the call
        ids = np.ascontiguousarray(np.asarray([int(x) for x in entry_ids], dtype=np.uint64))
        sch = (C.c_void_p * n)(*[_ptr(s) for _a, s in exported])
        arr = (C.c_void_p * n)(*[_ptr(a) for a, _s in exported])
        nh = N.HINT_SUBSTRING_SEARCH if hint == CacheExpression.SubstringSearch else (N.HINT_PREDICATE if hint else N.HINT_NONE)
        N.check(N.lib().lc_cache_insert_many(self._ctx, ids.ctypes.data, n, sch, arr, nh))
        for i, a in zip(ids, arrays):
            self._types[int(i)] = a.type

    def get(self, entry_id) -> Get:
        return Get(self, entry_id)

    def eval_predicate(self, entry_id, expr: LiquidExpr) -> EvaluatePredicate:
        return EvaluatePredicate(self, entry_id, expr)

    def is_cached(self, entry_id) -> bool:
        return bool(N.lib().lc_cache_is_cached(self._ctx, int(entry_id)))

    def try_read_liquid(self, entry_id) -> Optional[GpuLiquidArray]:
        # the reference hands out an Arc: the array stays alive (and unchanged) if the id is re-inserted, removed or the
        # cache reset while the caller holds it
        h = C.c_uint64(0)
        rc = N.lib().lc_cache_retain(self._ctx, int(entry_id), C.byref(h))
        if rc == N.LC_ERR_NOT_FOUND:
            return None
        N.check(rc)
        return GpuLiquidArray(self, int(h.value), owned=True)

    def remove(self, entry_id) -> bool:
        """Drop one entry (what eviction does to an in-memory entry, cache/core.rs:371-420); False when it was not cached.
        Arrays a caller still holds (`try_read_liquid`) keep working."""
        rc = N.lib().lc_cache_remove(self._ctx, int(entry_id))
        if rc == N.LC_ERR_NOT_FOUND:
            return False
        N.check(rc)
        self._types.pop(int(entry_id), None)
        return True

    def reset(self) -> None:
        N.check(N.lib().lc_cache_reset(self._ctx))
        self._types.clear()

    def stats(self) -> N.Stats:
        s = N.Stats()
        N.check(N.lib().lc_ctx_stats(self._ctx, C.byref(s)))
        return s

    def profile_counters(self, enable: bool) -> np.ndarray:
        """Measurement aid: returns the counters accumulated so far and switches accumulation on/off."""
        out = np.zeros(16, dtype=np.uint64)
        N.check(N.lib().lc_ctx_profile_counters(self._ctx, 1 if enable else 0, out.ctypes.data))
        return out

    def kernel_timing(self, enable: bool) -> None:
        N.check(N.lib().lc_ctx_kernel_timing(self._ctx, 1 if enable else 0))

    def last_kernel_ms(self) -> float:
        """Duration of the most recent predicate kernel (CUDA events recorded right around its launch)."""
        return float(N.lib().lc_ctx_last_kernel_ms(self._ctx))

    def set_stream(self, cuda_stream: int) -> None:
        N.check(N.lib().lc_ctx_set_stream(self._ctx, cuda_stream))

    def synchronize(self) -> None:
        N.check(N.lib().lc_ctx_synchronize(self._ctx))

    # -- LiquidArray-level helpers (transcode without the index) --
    def transcode(self, array: pa.Array, hint=None, compressor_scope: int = 0) -> GpuLiquidArray:
        """`transcode_liquid_inner_with_hint` (src/core/src/cache/transcode.rs:46-290)."""
        h = C.c_uint64(0)
        c_arr, c_sch = _export(array)
        nh = N.HINT_SUBSTRING_SEARCH if hint == CacheExpression.SubstringSearch else N.HINT_NONE
        N.check(N.lib().lc_encode(self._ctx, _ptr(c_sch), _ptr(c_arr), nh, compressor_scope, C.byref(h)))
        return GpuLiquidArray(self, int(h.value))

    def read_from_bytes(self, data: bytes, compressor_scope: Optional[int] = None) -> GpuLiquidArray:
        """`ipc::read_from_bytes` (liquid_array/ipc.rs:252-283): an LQDA image becomes an HBM-resident entry. Byte-view
        images need the scope whose symbol table they were compressed with (LiquidIPCContext)."""
        buf = np.frombuffer(data, dtype=np.uint8)
        h = C.c_uint64(0)
        if compressor_scope is None:
            N.check(N.lib().lc_from_bytes(self._ctx, buf.ctypes.data, len(buf), C.byref(h)))
        else:
            N.check(N.lib().lc_from_bytes_scoped(self._ctx, buf.ctypes.data, len(buf), int(compressor_scope), C.byref(h)))
        return GpuLiquidArray(self, int(h.value))

    def save_symbol_table(self, compressor_scope: int) -> bytes:
        """`save_symbol_table` (raw/fsst_buffer.rs:854-883) of the scope's FSST table."""
        nb = C.c_uint64(0)
        N.check(N.lib().lc_ctx_save_symbol_table(self._ctx, int(compressor_scope), None, 0, C.byref(nb)))
        buf = np.zeros(int(nb.value), dtype=np.uint8)
        N.check(N.lib().lc_ctx_save_symbol_table(self._ctx, int(compressor_scope), buf.ctypes.data, nb.value, C.byref(nb)))
        return buf.tobytes()

    def load_symbol_table(self, compressor_scope: int, data: bytes) -> None:
        """`load_symbol_table` (raw/fsst_buffer.rs:886-932): registers the table under a scope that has none."""
        buf = np.frombuffer(data, dtype=np.uint8)
        N.check(N.lib().lc_ctx_load_symbol_table(self._ctx, int(compressor_scope), buf.ctypes.data, len(buf)))

    def _handle(self, entry_id) -> int:
        ids = (C.c_uint64 * 1)(int(entry_id))
        out = (C.c_uint64 * 1)()
        N.check(N.lib().lc_cache_handles(self._ctx, ids, 1, out))
        return int(out[0])

    def handles(self, entry_ids: Sequence[int]) -> np.ndarray:
        ids = np.ascontiguousarray(np.asarray(entry_ids, dtype=np.uint64))
        out = np.zeros(len(ids), dtype=np.uint64)
        N.check(N.lib().lc_cache_handles(self._ctx, ids.ctypes.data, len(ids), out.ctypes.data))
        return out

    # -- batched forms (one launch sequence for many entries) --
    def eval_predicate_many(self, handles: np.ndarray, rows: np.ndarray, expr: LiquidExpr, column_type: pa.DataType,
                            selections: Optional[Sequence[Optional[np.ndarray]]] = None):
        """Returns (values bytes, validity bytes, byte_offsets, out_len, out_null_count, out_true_count)."""
        pred = expr.to_native(column_type)
        return self._eval_many_native(handles, rows, pred, selections)

    def _eval_many_native(self, handles, rows, pred, selections=None, out=None):
        n = len(handles)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        if out is None:
            sizes = (((np.asarray(rows, dtype=np.uint64) + 7) // 8 + 15) // 16) * 16
            offs = np.zeros(n, dtype=np.uint64)
            np.cumsum(sizes[:-1], out=offs[1:])
            total = int(sizes.sum())
            out = (np.zeros(total, dtype=np.uint8), np.zeros(total, dtype=np.uint8), offs,
                   np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64))
        vals, valid, offs, out_len, out_nulls = out[:5]
        true_counts = out[5] if len(out) > 5 else None
        sel_ptrs = None
        keep = None
        if selections is not None:
            keep = [s for s in selections]
            arr = (C.c_void_p * n)(*[(s.ctypes.data if s is not None else None) for s in keep])
            sel_ptrs = arr
        N.check(
            N.lib().lc_eval_predicate_many(
                self._ctx, handles.ctypes.data, n, C.byref(pred), sel_ptrs, vals.ctypes.data,
                valid.ctypes.data if valid is not None else None,  # NULL: the caller does not want validity (lc_gpu.h)
                offs.ctypes.data, out_len.ctypes.data, out_nulls.ctypes.data,
                true_counts.ctypes.data if true_counts is not None else None,
            )
        )
        return out

    def to_arrow_many(self, handles: np.ndarray, selections: Optional[Sequence[Optional[np.ndarray]]] = None) -> pa.Array:
        n = len(handles)
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        sel_ptrs = None
        if selections is not None:
            sel_ptrs = (C.c_void_p * n)(*[(s.ctypes.data if s is not None else None) for s in selections])
        out_a, out_s = _new_out()
        N.check(N.lib().lc_to_arrow_many(self._ctx, handles.ctypes.data, n, sel_ptrs, _ptr(out_s), _ptr(out_a)))
        return _import(out_a, out_s)

    def to_arrow_many_ptrs(self, handles: np.ndarray, sel_ptrs: np.ndarray) -> pa.Array:
        """to_arrow_many with the selections given as an array of host addresses (uint64; 0 = all rows)."""
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        sel_ptrs = np.ascontiguousarray(sel_ptrs, dtype=np.uint64)
        out_a, out_s = _new_out()
        N.check(N.lib().lc_to_arrow_many(self._ctx, handles.ctypes.data, len(handles), sel_ptrs.ctypes.data, _ptr(out_s), _ptr(out_a)))
        return _import(out_a, out_s)

    def and_then(self, left, right) -> pa.Array:
        """`boolean_buffer_and_then` (src/datafusion/src/utils.rs:62-83)."""
        lb, ln = selection_bits(left)
        rb, rn = selection_bits(right)
        out = np.zeros(len(lb) + 8, dtype=np.uint8)
        N.check(N.lib().lc_and_then(self._ctx, lb.ctypes.data, ln, rb.ctypes.data, rn, out.ctypes.data))
        return pa.array(np.unpackbits(out, bitorder="little")[:ln].astype(bool))

    def scan(self, rows_per_batch: Sequence[int]) -> "Scan":
        return Scan(self, rows_per_batch)


def or_terms(disjuncts) -> tuple[list, list, list]:
    """[[(handles, LiquidExpr, column_type), ...], ...] -> (handles per term, lowered predicates, disjunct per term), the
    arguments of `Scan.filter_or_native`. Raises UnsupportedExpr for a leaf `LiquidExpr.to_native` cannot lower."""
    if not disjuncts or any(len(d) == 0 for d in disjuncts):
        raise ValueError("filter_or: needs at least one disjunct, and at least one term in each")
    handles, preds, group = [], [], []
    for g, d in enumerate(disjuncts):
        for h, expr, typ in d:
            handles.append(h)
            preds.append(expr.to_native(typ))
            group.append(g)
    return handles, preds, group


def pack_or_terms(handles_per_term, preds, group, n_batches: int):
    """Checks the arguments of lc_scan_filter_or and packs them for ctypes: (pointer array of the handle lists, the arrays
    it points into, Predicate array, group array or None)."""
    n = len(preds)
    if n == 0:
        raise ValueError("filter_or: no terms")
    if len(handles_per_term) != n:
        raise ValueError(f"filter_or: {len(handles_per_term)} handle lists for {n} predicates")
    keep = [np.ascontiguousarray(h, dtype=np.uint64) for h in handles_per_term]
    for t, h in enumerate(keep):
        if h.ndim != 1 or len(h) != n_batches:
            raise ValueError(f"filter_or: term {t} has {h.size} handles, the scan has {n_batches} batches")
    g_arr = None
    if group is not None:
        g = [int(x) for x in group]
        if len(g) != n:
            raise ValueError(f"filter_or: {len(g)} group indices for {n} terms")
        if g[0] != 0 or any(b - a not in (0, 1) for a, b in zip(g, g[1:])):
            raise ValueError("filter_or: group must start at 0 and be non-decreasing without gaps")
        g_arr = (C.c_uint32 * n)(*g)
    h_ptrs = (C.c_void_p * n)(*[h.ctypes.data for h in keep])
    p_arr = (N.Predicate * n)(*preds)
    keep.append(list(preds))  # the literal bytes the copied structs point at
    return h_ptrs, keep, p_arr, g_arr


class Scan:
    """The per-batch loop of `LiquidCacheReader::build_predicate_filter` + `read_from_cache`
    (/root/reference/src/datafusion/src/reader/runtime/liquid_cache_reader.rs:297-391) for many batches at
    once, with the running selection resident in HBM between conjuncts."""

    def __init__(self, cache: LiquidCache, rows_per_batch: Sequence[int]):
        self._cache = cache
        self._rows = np.ascontiguousarray(np.asarray(rows_per_batch, dtype=np.uint64))
        self._scan = C.c_void_p()
        N.check(N.lib().lc_scan_begin(cache._ctx, len(self._rows), self._rows.ctypes.data, C.byref(self._scan)))

    def close(self):
        if self._scan:
            N.lib().lc_scan_end(self._scan)
            self._scan = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self) -> None:
        N.check(N.lib().lc_scan_reset(self._scan))

    def set_selection(self, batch: int, selection) -> None:
        bits, n = selection_bits(selection)
        N.check(N.lib().lc_scan_set_selection(self._scan, batch, bits.ctypes.data, n))

    def selection_layout(self) -> tuple[np.ndarray, int]:
        """(word offset of every batch, total words) of the running selection as store / load move it."""
        offs = np.zeros(len(self._rows), dtype=np.uint64)
        tot = C.c_uint64(0)
        N.check(N.lib().lc_scan_selection_layout(self._scan, offs.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(tot)))
        return offs, int(tot.value)

    def store_selections(self) -> np.ndarray:
        """The running selection of every batch in one download (uint32 words, LSB first, layout: selection_layout)."""
        _offs, tot = self.selection_layout()
        out = np.zeros(tot, dtype=np.uint32)
        N.check(N.lib().lc_scan_store_selections(self._scan, out.ctypes.data, tot))
        return out

    def load_selections(self, words: np.ndarray) -> None:
        words = np.ascontiguousarray(words, dtype=np.uint32)
        N.check(N.lib().lc_scan_load_selections(self._scan, words.ctypes.data, len(words)))

    def filter(self, handles: np.ndarray, expr: LiquidExpr, column_type: pa.DataType) -> None:
        pred = expr.to_native(column_type)
        self.filter_native(handles, pred)

    def filter_native(self, handles: np.ndarray, pred: N.Predicate) -> None:
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        N.check(N.lib().lc_scan_filter(self._scan, handles.ctypes.data, C.byref(pred)))

    def filter_or(self, disjuncts) -> None:
        """One conjunct that is an OR of AND groups: `disjuncts` = [[(handles, LiquidExpr, column_type), ...], ...];
        selection &= OR over the groups of (AND over the group's terms). Every leaf is lowered like `filter` lowers it."""
        self.filter_or_native(*or_terms(disjuncts))

    def filter_or_native(self, handles_per_term, preds, group=None) -> None:
        """lc_scan_filter_or: `handles_per_term[t]` the batch handles of term t, `preds[t]` its lowered predicate,
        `group[t]` its disjunct (non-decreasing from 0, no gaps; None = every term its own disjunct)."""
        h_ptrs, keep, p_arr, g_arr = pack_or_terms(handles_per_term, preds, group, len(self._rows))
        N.check(N.lib().lc_scan_filter_or(self._scan, len(preds), h_ptrs, p_arr, g_arr))
        del keep

    def counts(self) -> tuple[np.ndarray, int]:
        out = np.zeros(len(self._rows), dtype=np.uint64)
        tot = C.c_uint64(0)
        N.check(N.lib().lc_scan_counts(self._scan, out.ctypes.data, C.byref(tot)))
        return out, int(tot.value)

    def selection(self, batch: int) -> pa.Array:
        rows = int(self._rows[batch])
        out = np.zeros((rows + 7) // 8 + 8, dtype=np.uint8)
        N.check(N.lib().lc_scan_selection(self._scan, batch, out.ctypes.data))
        return pa.array(np.unpackbits(out, bitorder="little")[:rows].astype(bool))

    def read(self, handles: np.ndarray) -> pa.Array:
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        out_a, out_s = _new_out()
        N.check(N.lib().lc_scan_read(self._scan, handles.ctypes.data, _ptr(out_s), _ptr(out_a)))
        return _import(out_a, out_s)

    def read_device(self, handles: np.ndarray, d_values: int = 0, values_cap: int = 0, d_offsets: int = 0,
                    d_validity: int = 0) -> tuple[int, int, int]:
        """lc_scan_read_device: the concatenated result stays in CALLER-owned device memory (raw device addresses;
        e.g. torch tensors' data_ptr()). All pointers 0 = size query. Returns (rows, value_bytes, null_count).
        Buffers: values `value_bytes`; offsets (byte-view) `4 * (rows + 1)`; validity `4 * ceil(rows / 32)`."""
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        rows, nbytes, nulls = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        N.check(N.lib().lc_scan_read_device(self._scan, handles.ctypes.data, d_values or None, values_cap, d_offsets or None,
                                            d_validity or None, C.byref(rows), C.byref(nbytes), C.byref(nulls)))
        return int(rows.value), int(nbytes.value), int(nulls.value)

    def read_async(self, handles: np.ndarray, d_values: int, values_cap: int, d_offsets: int, rows_cap: int, d_header: int) -> bool:
        """lc_scan_read_async: enqueue the device-planned read of the column into caller-owned device buffers (raw device
        addresses) and return without synchronising; the 64-byte header (rows at byte 8, value bytes at 16, overflow at 4)
        lands at `d_header`. False when this column is not read by the device-planned path."""
        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        rc = N.lib().lc_scan_read_async(self._scan, handles.ctypes.data, d_values, values_cap, d_offsets or None, rows_cap, d_header)
        if rc == N.LC_ERR_UNSUPPORTED_EXPR:
            return False
        N.check(rc)
        return True

    def read_torch_borrowed(self, handles: np.ndarray, device):
        """The filtered column as torch tensors over the scan's OWN device buffer (lc_scan_read_borrowed: planned on the
        device, one synchronisation, nothing but a 64-byte header crosses PCIe): `(values u8[value_bytes], offsets
        i32[rows+1] | None, rows)`, valid until the next read on this scan. None when this read cannot be planned on the
        device (first read of a scan, nulls, unsupported type): use `read_torch`."""
        import torch

        handles = np.ascontiguousarray(handles, dtype=np.uint64)
        dv, do = C.c_void_p(), C.c_void_p()
        rows, nbytes = C.c_uint64(0), C.c_uint64(0)
        rc = N.lib().lc_scan_read_borrowed(self._scan, handles.ctypes.data, C.byref(dv), C.byref(do), C.byref(rows), C.byref(nbytes))
        if rc == N.LC_ERR_UNSUPPORTED_EXPR:
            return None
        N.check(rc)

        class _Dev:  # __cuda_array_interface__ over a raw device range: torch.as_tensor wraps it without copying
            def __init__(self, ptr, n, typestr):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}

        nb, nr = int(nbytes.value), int(rows.value)
        values = torch.as_tensor(_Dev(dv.value, nb, "|u1"), device=device) if nb else torch.empty(0, dtype=torch.uint8, device=device)
        offsets = torch.as_tensor(_Dev(do.value, nr + 1, "<i4"), device=device) if do.value else None
        return values, offsets, nr

    def read_torch(self, handles: np.ndarray, device):
        """read_device into freshly allocated torch tensors on `device`:
        (values u8[value_bytes], offsets i32[rows+1] | None, validity u8[4*ceil(rows/32)] | None, rows, null_count)."""
        import torch

        rows, nbytes, nulls = self.read_device(handles)
        is_bytes = int(N.lib().lc_data_type(self._cache._ctx, int(handles[0]))) == N.LIQUID_BYTE_VIEW
        values = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
        offsets = torch.empty(rows + 1, dtype=torch.int32, device=device) if is_bytes else None
        validity = torch.empty(4 * ((rows + 31) // 32), dtype=torch.uint8, device=device) if nulls else None
        self.read_device(handles, values.data_ptr(), nbytes, offsets.data_ptr() if offsets is not None else 0,
                         validity.data_ptr() if validity is not None else 0)
        return values[:nbytes], offsets, validity, rows, nulls
