"""Host-side mirror of the predicate shapes the reference admits.

Reference: `LiquidExpr::try_new` / `supports_expr` (/root/reference/src/core/src/cache/liquid_expr.rs:33-202)
and `ByteViewExpression::try_from` (src/core/src/liquid_array/byte_view_array/operator.rs:134-176).
The reference receives DataFusion `PhysicalExpr` trees; these small classes are the same trees with the
same names, so parity tests read like the reference's. `LiquidExpr.to_native()` lowers a validated
expression to the `lc_predicate` struct of the C ABI (op + typed literal) — planning only, no data touched.
"""
from __future__ import annotations

import datetime as _dt
from dataclasses import dataclass
from typing import Any, Optional

import numpy as _np
import pyarrow as pa

from . import _native as N


# ---- PhysicalExpr node mirrors (datafusion_physical_expr::expressions) ----
@dataclass(frozen=True)
class Column:
    name: str
    index: int = 0


@dataclass(frozen=True)
class Literal:
    """`Literal(ScalarValue)`; `value` is a Python int / str / bytes / bool / date / None."""

    value: Any
    data_type: Optional[pa.DataType] = None


@dataclass(frozen=True)
class BinaryExpr:
    left: Any
    op: str  # "=", "!=", "<", "<=", ">", ">=", "LikeMatch", "NotLikeMatch", or anything else (unsupported)
    right: Any


@dataclass(frozen=True)
class LikeExpr:
    negated: bool
    case_insensitive: bool
    expr: Any
    pattern: Any


@dataclass(frozen=True)
class InListExpr:
    """`InListExpr { expr, list, negated }`: `expr [NOT] IN (list)`. The reference's LiquidExpr does not admit it
    (`try_new` returns None); `LiquidExpr.new_unchecked(InListExpr(...))` lowers it to LC_OP_IN / LC_OP_NOT_IN."""

    expr: Any
    list: tuple
    negated: bool = False


@dataclass(frozen=True)
class CastExpr:
    expr: Any
    cast_type: Optional[pa.DataType] = None


CastColumnExpr = CastExpr
TryCastExpr = CastExpr


@dataclass(frozen=True)
class ScalarFunctionExpr:
    name: str
    args: tuple


@dataclass(frozen=True)
class DynamicFilterPhysicalExpr:
    current: Any  # the expression `dynamic_filter.current()` returns


class CacheExpression:
    """`CacheExpression` hints (src/core/src/cache/expressions.rs:38-53)."""

    SubstringSearch = "SubstringSearch"
    PredicateColumn = "PredicateColumn"

    @staticmethod
    def substring_search():
        return CacheExpression.SubstringSearch

    @staticmethod
    def extract_date32(field: str):
        """`CacheExpression::extract_date32(Date32Field)` (expressions.rs:82-84); field in Year / Month / Day / DayOfWeek."""
        assert field in ("Year", "Month", "Day", "DayOfWeek")
        return ("ExtractDate32", field)

    @staticmethod
    def as_date32_field(hint):
        """`as_date32_field` (expressions.rs:133-138)"""
        return hint[1] if isinstance(hint, tuple) and hint[0] == "ExtractDate32" else None


_CMP_OPS = {"=": N.OP_EQ, "!=": N.OP_NE, "<": N.OP_LT, "<=": N.OP_LE, ">": N.OP_GT, ">=": N.OP_GE}


def is_byte_like(t: pa.DataType) -> bool:
    if pa.types.is_dictionary(t):
        return is_byte_like(t.value_type)
    return (
        pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_string_view(t) or pa.types.is_binary_view(t)
    )


def is_numeric_like(t: pa.DataType) -> bool:
    if pa.types.is_timestamp(t):
        return t.tz is None
    return (
        pa.types.is_integer(t)
        or pa.types.is_floating(t)
        or pa.types.is_date(t)
        or pa.types.is_decimal(t)
    )


def _is_column_like(e) -> bool:
    if isinstance(e, Column):
        return True
    if isinstance(e, CastExpr):
        return _is_column_like(e.expr)
    return False


def _is_to_timestamp_seconds_column(e) -> bool:
    return isinstance(e, ScalarFunctionExpr) and e.name == "to_timestamp_seconds" and len(e.args) == 1 and _is_column_like(e.args[0])


def _bytes_needle(lit: Literal) -> Optional[bytes]:
    """get_bytes_needle (src/core/src/utils/mod.rs:34-46)."""
    v = lit.value
    if isinstance(v, str):
        return v.encode("utf-8")
    if isinstance(v, (bytes, bytearray)):
        return bytes(v)
    return None


class LiquidExpr:
    """A predicate expression validated for LiquidCache predicate evaluation."""

    def __init__(self, expr):
        self._expr = expr

    @staticmethod
    def try_new(expr, data_type: pa.DataType, expression_hint=None) -> Optional["LiquidExpr"]:
        if isinstance(expr, DynamicFilterPhysicalExpr):
            expr = expr.current
            if expr is None:
                return None
        return LiquidExpr(expr) if _supports_expr(expr, data_type, expression_hint) else None

    @staticmethod
    def new_unchecked(expr) -> "LiquidExpr":
        return LiquidExpr(expr)

    def physical_expr(self):
        return self._expr

    def __repr__(self):
        return f"LiquidExpr({self._expr!r})"

    # ---- lowering to the C ABI ----
    def to_native(self, column_type: pa.DataType) -> N.Predicate:
        e = self._expr
        if isinstance(e, DynamicFilterPhysicalExpr):
            e = e.current
        p = N.Predicate()
        if isinstance(e, Literal) and isinstance(e.value, bool):
            p.op = N.OP_CONST_TRUE if e.value else N.OP_CONST_FALSE
            return p
        if isinstance(e, LikeExpr):
            if e.case_insensitive or not isinstance(e.pattern, Literal):
                raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "ILIKE / non-literal pattern")
            needle = _bytes_needle(e.pattern)
            if needle is None:
                raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "LIKE pattern is not bytes-like")
            p.op = N.OP_NOT_LIKE if e.negated else N.OP_LIKE
            _set_bytes(p, needle)
            return p
        if isinstance(e, BinaryExpr) and isinstance(e.right, Literal):
            if e.op in ("LikeMatch", "NotLikeMatch"):
                needle = _bytes_needle(e.right)
                if needle is None:
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "LIKE pattern is not bytes-like")
                p.op = N.OP_LIKE if e.op == "LikeMatch" else N.OP_NOT_LIKE
                _set_bytes(p, needle)
                return p
            if e.op not in _CMP_OPS:
                raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, f"operator {e.op}")
            p.op = _CMP_OPS[e.op]
            if is_byte_like(column_type):
                needle = _bytes_needle(e.right)
                if needle is None:
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal is not bytes-like")
                _set_bytes(p, needle)
                return p
            if pa.types.is_floating(column_type):
                # Float32/Float64 columns: the literal DataFusion hands over has the column's type; it crosses
                # the ABI as f64 bits (exact for either width)
                if not isinstance(e.left, Column):
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "float column under a cast")
                v = e.right.value
                if isinstance(v, bool) or not isinstance(v, (int, float)):
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal is not a float")
                if pa.types.is_float32(column_type):
                    v = float(_np.float32(v))
                p.lit_kind = N.LIT_F64
                p.lit_u64 = int(_np.array([float(v)], dtype=_np.float64).view(_np.uint64)[0])
                return p
            if pa.types.is_decimal(column_type):
                # Decimal128/256: unscaled integer at the column's scale (the coerced ScalarValue::Decimal128)
                if not isinstance(e.left, Column):
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "decimal column under a cast")
                u = _decimal_unscaled(e.right.value, column_type.scale)
                if u is not None and pa.types.is_decimal256(column_type) and not (-(1 << 127) <= u < (1 << 127)) and -(1 << 255) <= u < (1 << 255):
                    _set_bytes(p, (u & ((1 << 256) - 1)).to_bytes(32, "little"))  # the column's own little-endian integer
                    return p
                if u is None or not (-(1 << 127) <= u < (1 << 127)):
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal is not a decimal at the column's scale")
                p.lit_kind = N.LIT_I128
                p.lit_u64 = u & 0xFFFFFFFFFFFFFFFF
                hi = (u >> 64) & 0xFFFFFFFFFFFFFFFF
                p.lit_i64 = hi - (1 << 64) if hi >= (1 << 63) else hi
                return p
            if not _cast_chain_is_integer_identity(e.left, column_type):
                # e.g. to_timestamp_seconds(col) or a narrowing cast: the reference evaluates these with
                # DataFusion on the decoded array; the caller keeps doing that.
                raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "column side is not an integer-preserving cast chain")
            v = _int_literal(e.right, _outermost_type(e.left, column_type))
            if v is None:
                raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal is not an integer/date/timestamp")
            if v < 0 or v <= 0x7FFFFFFFFFFFFFFF:
                if v < -(1 << 63):
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal out of i64 range")
                p.lit_kind = N.LIT_I64
                p.lit_i64 = v
            else:
                if v > 0xFFFFFFFFFFFFFFFF:
                    raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, "literal out of u64 range")
                p.lit_kind = N.LIT_U64
                p.lit_u64 = v
            return p
        if isinstance(e, InListExpr):
            return _lower_in_list(e, column_type)
        raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, f"expression shape {type(e).__name__}")


def _lower_in_list(e: "InListExpr", column_type: pa.DataType) -> N.Predicate:
    """`col [NOT] IN (v1, ..., vn)` -> LC_OP_IN / LC_OP_NOT_IN. The column side follows the rules of a comparison; the
    values are n little-endian 8-byte integers (LC_LIT_I64, or LC_LIT_U64 when one exceeds i64) or, on byte-like columns,
    Arrow's Utf8 layout (int32 offsets[n + 1], then the bytes). Null or non-literal elements are refused."""
    def refuse(why):
        raise N.UnsupportedExpr(N.LC_ERR_UNSUPPORTED_EXPR, why)

    p = N.Predicate()
    p.op = N.OP_NOT_IN if e.negated else N.OP_IN
    items = list(e.list)
    for it in items:
        if not isinstance(it, Literal) or it.value is None:
            refuse("IN list element is not a non-null literal")
    if is_byte_like(column_type):
        if not _is_column_like(e.expr):
            refuse("IN list: column side is not column-like")
        needles = [_bytes_needle(it) for it in items]
        if any(nd is None for nd in needles):
            refuse("IN list element is not bytes-like")
        offs = _np.zeros(len(needles) + 1, dtype="<i4")
        offs[1:] = _np.cumsum([len(nd) for nd in needles], dtype=_np.int64) if needles else []
        _set_bytes(p, offs.tobytes() + b"".join(needles))
        p.lit_len = len(needles)
        return p
    if pa.types.is_floating(column_type) or pa.types.is_decimal(column_type):
        refuse("IN list on a float / decimal column")
    if not _cast_chain_is_integer_identity(e.expr, column_type):
        refuse("IN list: column side is not an integer-preserving cast chain")
    outer = _outermost_type(e.expr, column_type)
    vals = []
    for it in items:
        v = _int_literal(it, outer)
        if v is None:
            refuse("IN list element is not an integer/date/timestamp")
        if not (-(1 << 63) <= v <= 0xFFFFFFFFFFFFFFFF):
            refuse("IN list element out of the 64-bit range")
        vals.append(v)
    if any(v > 0x7FFFFFFFFFFFFFFF for v in vals):
        if any(v < 0 for v in vals):
            refuse("IN list mixes negative values with values above i64")
        p.lit_kind = N.LIT_U64
        raw = _np.array(vals, dtype="<u8").tobytes()
    else:
        p.lit_kind = N.LIT_I64
        raw = _np.array(vals, dtype="<i8").tobytes()
    p._keepalive = raw
    p.lit_bytes = raw
    p.lit_len = len(vals)
    return p


def _set_bytes(p: N.Predicate, needle: bytes) -> None:
    p.lit_kind = N.LIT_BYTES
    p._keepalive = needle  # ctypes does not keep the bytes object alive by itself
    p.lit_bytes = needle
    p.lit_len = len(needle)


def _decimal_unscaled(v, scale: int) -> Optional[int]:
    """Unscaled integer of a decimal literal at `scale`; None when the value has more fractional digits."""
    import decimal as _dec

    if isinstance(v, bool):
        return None
    if isinstance(v, int):
        d = _dec.Decimal(v)
    elif isinstance(v, _dec.Decimal):
        d = v
    else:
        return None
    with _dec.localcontext() as cx:
        cx.prec = 100
        scaled = d.scaleb(scale)
        if scaled != scaled.to_integral_value():
            return None
        return int(scaled)


def _int_literal(lit: Literal, compared_type: Optional[pa.DataType] = None) -> Optional[int]:
    """The literal in the integer domain of `compared_type` (the column's type, or the outermost cast's): a
    `datetime.date` is a day count against Date32 and milliseconds against Date64 — the two physical units the reference's
    Date32 / Date64 primitive arrays hold (primitive_array.rs:55-68)."""
    v = lit.value
    if isinstance(v, bool):
        return None
    if isinstance(v, int):
        return v
    if isinstance(v, _dt.datetime):
        return None
    if isinstance(v, _dt.date):
        days = (v - _dt.date(1970, 1, 1)).days
        if compared_type is not None and pa.types.is_date64(compared_type):
            return days * 86_400_000
        if compared_type is None or pa.types.is_date32(compared_type) or pa.types.is_integer(compared_type):
            return days
        return None  # a date against a timestamp column: DataFusion would have coerced it to a timestamp literal
    return None


def _int_range(t: pa.DataType):
    """Value range of an integer-like type in its own integer domain, None when casts from/to it rescale."""
    if pa.types.is_integer(t):
        bits = t.bit_width
        return (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if pa.types.is_signed_integer(t) else (0, (1 << bits) - 1)
    if pa.types.is_date32(t):
        return (-(1 << 31), (1 << 31) - 1)
    return None


def _outermost_type(e, column_type: pa.DataType) -> pa.DataType:
    return e.cast_type if isinstance(e, CastExpr) and e.cast_type is not None else column_type


def _cast_chain_is_integer_identity(e, column_type: pa.DataType) -> bool:
    """Column possibly under casts that keep the integer value for EVERY value of the source type (e.g. UInt16 -> Int32 ->
    Date32 for ClickBench's "EventDate"::INT::DATE). A narrowing or sign-changing cast (Int64 -> Int8, UInt64 -> Int64) is
    not one: DataFusion's cast gives an error or a null for the values that do not fit, so the caller keeps evaluating
    those on the decoded array, like every cast that rescales (Date64 -> Date32, timestamps)."""
    chain = []
    while isinstance(e, CastExpr):
        chain.append(e.cast_type)
        e = e.expr
    if not isinstance(e, Column):
        return False
    if not chain:
        return (pa.types.is_integer(column_type) or pa.types.is_date(column_type)
                or (pa.types.is_timestamp(column_type) and column_type.tz is None))
    src = _int_range(column_type)
    if src is None:
        return False
    for t in reversed(chain):  # innermost cast first
        if t is None:
            continue
        dst = _int_range(t)
        if dst is None or dst[0] > src[0] or dst[1] < src[1]:
            return False
        src = dst
    return True


def _column_name(e) -> Optional[str]:
    """The column under a cast chain (CastExpr / CastColumnExpr / TryCastExpr), None for anything else."""
    while isinstance(e, CastExpr):
        e = e.expr
    return e.name if isinstance(e, Column) else None


def _column_literal_leaf(e) -> Optional[str]:
    """`extract_column_literal` (src/datafusion/src/reader/runtime/liquid_predicate.rs:45-68) for the leaves this library
    lowers: a column (or a cast chain over one) compared with a literal, LIKE / NOT LIKE against a literal pattern, or an
    IN list. Returns the column's name."""
    if isinstance(e, BinaryExpr) and isinstance(e.right, Literal) and (e.op in _CMP_OPS or e.op in ("LikeMatch", "NotLikeMatch")):
        return _column_name(e.left)
    if isinstance(e, LikeExpr) and isinstance(e.pattern, Literal):
        return _column_name(e.expr)
    if isinstance(e, InListExpr):
        return _column_name(e.expr)
    return None


def split_disjunction(expr) -> Optional[list]:
    """An OR of column-literal leaves, or of AND groups of them, as `[[(column_name, leaf), ...], ...]` (one inner list per
    disjunct, in the tree's left-to-right order) for `Scan.filter_or`; None for any other tree. The pure-OR case is
    `extract_multi_column_or` (liquid_predicate.rs:12-43): the top node must be an OR, so there are at least two leaves.
    AND is never distributed over OR: an AND group must hold leaves (or nested ANDs of leaves) only."""
    if isinstance(expr, DynamicFilterPhysicalExpr):
        expr = expr.current
    if not (isinstance(expr, BinaryExpr) and expr.op == "OR"):
        return None

    def disjuncts(e, out) -> bool:
        if isinstance(e, BinaryExpr) and e.op == "OR":
            return disjuncts(e.left, out) and disjuncts(e.right, out)
        group = []
        if not conjuncts(e, group):
            return False
        out.append(group)
        return True

    def conjuncts(e, out) -> bool:
        if isinstance(e, BinaryExpr) and e.op == "AND":
            return conjuncts(e.left, out) and conjuncts(e.right, out)
        name = _column_literal_leaf(e)
        if name is None:
            return False
        out.append((name, e))
        return True

    out: list = []
    return out if disjuncts(expr, out) else None


def _supports_expr(expr, data_type, hint) -> bool:
    if isinstance(expr, BinaryExpr):
        return _supports_binary_expr(expr, data_type, hint)
    if isinstance(expr, LikeExpr):
        return _supports_like_expr(expr, data_type, hint)
    if isinstance(expr, Literal):
        return isinstance(expr.value, bool) and is_byte_like(data_type)
    return False


def _supports_binary_expr(b: BinaryExpr, data_type, hint) -> bool:
    if not isinstance(b.right, Literal):
        return False
    if is_byte_like(data_type):
        if not _is_column_like(b.left):
            return False
        if b.op in _CMP_OPS:
            return _bytes_needle(b.right) is not None
        if b.op in ("LikeMatch", "NotLikeMatch"):
            return _bytes_needle(b.right) is not None and hint == CacheExpression.SubstringSearch
        return False
    if is_numeric_like(data_type):
        return b.op in _CMP_OPS and (_is_column_like(b.left) or _is_to_timestamp_seconds_column(b.left))
    return False


def _supports_like_expr(l: LikeExpr, data_type, hint) -> bool:
    if not is_byte_like(data_type) or l.case_insensitive:
        return False
    if not _is_column_like(l.expr) or hint != CacheExpression.SubstringSearch:
        return False
    return isinstance(l.pattern, Literal) and _bytes_needle(l.pattern) is not None
