"""`col [NOT] IN (list)` without a GPU: the integer kernels' list planner (int_plan.cuh plan_int_in, compiled for the host by
tests/cpp/in_list_plan_host.cc) against brute-force membership, the lowering of InListExpr to the C ABI
(LiquidExpr.to_native), and the two new op values of include/lc_gpu.h."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pyarrow as pa
import pytest

from liquid_cache_b200 import _native as N
from liquid_cache_b200.expr import CastExpr, Column, InListExpr, LiquidExpr, Literal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_pins_the_in_ops_and_caps():
    text = open(os.path.join(ROOT, "include", "lc_gpu.h")).read()
    assert int(re.search(r"LC_OP_IN\s*=\s*(\d+)", text).group(1)) == N.OP_IN == 10
    assert int(re.search(r"LC_OP_NOT_IN\s*=\s*(\d+)", text).group(1)) == N.OP_NOT_IN == 11
    assert int(re.search(r"#define LC_IN_LIST_MAX_VALUES (\d+)", text).group(1)) == N.IN_LIST_MAX_VALUES >= 256
    assert int(re.search(r"#define LC_IN_LIST_MAX_BYTES (\d+)", text).group(1)) == N.IN_LIST_MAX_BYTES >= 16384


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "build", "tests", "libin_list_plan_host.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-Wno-unused-function", "-shared", "-fPIC", f"-I{ROOT}",
                        "-I/usr/local/cuda/include", os.path.join(ROOT, "tests", "cpp", "in_list_plan_host.cc"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    l = C.CDLL(out)
    l.ilp_eval.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_uint32,
                           C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    return l


def plan_eval(lib, tbits, width, signed, reference, values, offs, negated):
    """values: the list as Python ints in the column's domain; offs: packed values. Returns (mask, shape)."""
    vals = sorted(set(values))
    words = np.array([v & 0xFFFFFFFFFFFFFFFF for v in vals], dtype=np.uint64)
    packed = np.ascontiguousarray(offs, dtype=np.uint64)
    out = np.zeros(len(packed), dtype=np.uint8)
    a, b = C.c_uint32(0), C.c_uint32(0)
    shape = lib.ilp_eval(tbits, width, int(signed), reference & ((1 << tbits) - 1), words.ctypes.data if len(words) else None, len(words),
                         int(negated), packed.ctypes.data, len(packed), out.ctypes.data, C.byref(a), C.byref(b))
    return out.astype(bool), shape


@pytest.mark.parametrize("np_dt", [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64], ids=lambda d: np.dtype(d).name)
def test_planner_matches_brute_force_membership(lib, np_dt):
    info = np.iinfo(np_dt)
    tbits, signed = info.bits, info.min < 0
    rng = np.random.default_rng(1000 + tbits + signed)
    widths = sorted({1, 2, 3, 7, tbits // 2, tbits - 1, tbits} | ({31, 32, 33, 63} if tbits == 64 else set()))
    shapes = set()
    for width in widths:
        span = (1 << width) - 1
        refs = {info.min, info.max - span, 0 if not signed else -5, max(info.min, min(info.max - span, 1000))}
        for reference in refs:
            if reference < info.min or reference + span > info.max:
                continue
            offs = np.unique(np.concatenate([rng.integers(0, span, size=150, endpoint=True, dtype=np.uint64),
                                             np.array([0, span, span // 2], dtype=np.uint64)]))
            window = [reference + int(o) for o in offs]
            for trial in range(8):
                k = int(rng.integers(0, 40))
                picks = [int(x) for x in rng.choice(window, size=min(k, len(window)))] if k else []
                extra = [reference - 1, reference + span + 1, info.min, info.max, reference, reference + span]
                if trial % 2:
                    extra += [reference + 3, reference + 4, reference + 5]  # a consecutive run
                lst = picks + [e for e in extra[: trial] if info.min <= e <= info.max]
                if trial == 0:
                    lst = []
                if trial == 1 and window:
                    lst = [window[len(window) // 2]] * 3  # duplicates of one value
                for negated in (False, True):
                    got, shape = plan_eval(lib, tbits, width, signed, reference, lst, offs, negated)
                    s = set(lst)
                    want = np.array([(v in s) != negated for v in window])
                    assert np.array_equal(got, want), (np.dtype(np_dt).name, width, reference, sorted(s), negated)
                    shapes.add(shape)
    assert shapes == {0, 1, 2}


def test_single_values_and_runs_lower_to_a_range(lib):
    offs = np.arange(0, 64, dtype=np.uint64)
    for lst in ([10], [10, 11, 12], [5, 6, 7, 8, 9]):
        got, shape = plan_eval(lib, 32, 6, False, 0, lst, offs, False)
        assert shape == 1 and np.array_equal(got, np.isin(offs, lst))
    got, shape = plan_eval(lib, 32, 6, False, 0, [3, 9], offs, False)
    assert shape == 2 and np.array_equal(got, np.isin(offs, [3, 9]))
    got, shape = plan_eval(lib, 32, 6, False, 100, [1, 2], offs, True)  # nothing in the window: NOT IN is true
    assert shape == 0 and got.all()


# ---- to_native lowering ----
def _lower(expr, typ):
    return LiquidExpr.new_unchecked(expr).to_native(typ)


def _at(p, n):
    """n bytes at the predicate's lit_bytes pointer (the field itself reads back as a NUL-terminated copy)"""
    addr = C.c_void_p.from_buffer(p, N.Predicate.lit_bytes.offset).value
    return C.string_at(addr, n)


def _raw(p):
    return _at(p, 8 * p.lit_len)


def test_integer_lists_lower_to_i64_words():
    p = _lower(InListExpr(Column("c"), (Literal(-1), Literal(6), Literal(6))), pa.int16())
    assert (p.op, p.lit_kind, p.lit_len) == (N.OP_IN, N.LIT_I64, 3)
    assert np.frombuffer(_raw(p), dtype="<i8").tolist() == [-1, 6, 6]
    p = _lower(InListExpr(Column("c"), (Literal(1),), negated=True), pa.uint8())
    assert (p.op, p.lit_kind) == (N.OP_NOT_IN, N.LIT_I64)


def test_values_above_i64_lower_to_u64_words():
    big = 2**63 + 5
    p = _lower(InListExpr(Column("c"), (Literal(big), Literal(3))), pa.uint64())
    assert p.lit_kind == N.LIT_U64 and np.frombuffer(_raw(p), dtype="<u8").tolist() == [big, 3]
    with pytest.raises(N.UnsupportedExpr):
        _lower(InListExpr(Column("c"), (Literal(big), Literal(-3))), pa.uint64())


def test_dates_and_integer_identity_casts_lower():
    import datetime as dt

    p = _lower(InListExpr(CastExpr(CastExpr(Column("EventDate"), pa.int32()), pa.date32()), (Literal(dt.date(2013, 7, 15)),)), pa.uint16())
    assert np.frombuffer(_raw(p), dtype="<i8").tolist() == [(dt.date(2013, 7, 15) - dt.date(1970, 1, 1)).days]
    p = _lower(InListExpr(Column("d"), (Literal(dt.date(1970, 1, 2)),)), pa.date64())
    assert np.frombuffer(_raw(p), dtype="<i8").tolist() == [86_400_000]
    with pytest.raises(N.UnsupportedExpr):
        _lower(InListExpr(CastExpr(Column("c"), pa.int8()), (Literal(1),)), pa.int64())  # narrowing cast


def test_byte_lists_lower_to_the_utf8_layout():
    p = _lower(InListExpr(Column("s"), (Literal("MAIL"), Literal(b"SHIP"), Literal(""))), pa.string())
    assert (p.op, p.lit_kind, p.lit_len) == (N.OP_IN, N.LIT_BYTES, 3)
    raw = _at(p, 16 + 8)
    assert np.frombuffer(raw[:16], dtype="<i4").tolist() == [0, 4, 8, 8] and raw[16:] == b"MAILSHIP"
    p = _lower(InListExpr(Column("s"), ()), pa.dictionary(pa.uint16(), pa.utf8()))
    assert p.lit_len == 0 and _at(p, 4) == b"\0\0\0\0"


@pytest.mark.parametrize("expr,typ", [
    (InListExpr(Column("c"), (Literal(1), Literal(None))), pa.int32()),
    (InListExpr(Column("c"), (Literal(1), Column("d"))), pa.int32()),
    (InListExpr(Column("c"), (Literal(1.5),)), pa.float64()),
    (InListExpr(Column("c"), (Literal(1),)), pa.float32()),
    (InListExpr(Column("c"), (Literal(1),)), pa.decimal128(10, 2)),
    (InListExpr(Column("s"), (Literal("a"), Literal(None))), pa.string()),
    (InListExpr(Column("s"), (Literal(3),)), pa.string()),
], ids=["null", "non-literal", "float-list", "float-col", "decimal", "null-bytes", "int-on-bytes"])
def test_refusals(expr, typ):
    with pytest.raises(N.UnsupportedExpr):
        _lower(expr, typ)


def test_try_new_keeps_refusing_in_lists():
    for typ in (pa.int32(), pa.string(), pa.date32()):
        assert LiquidExpr.try_new(InListExpr(Column("c"), (Literal(1),)), typ) is None
        assert LiquidExpr.try_new(InListExpr(Column("c"), (Literal("a"),), negated=True), typ) is None
