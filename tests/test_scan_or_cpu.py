"""CPU side of lc_scan_filter_or (Scan.filter_or): splitting an OR tree into disjuncts (the reference's
extract_multi_column_or, src/datafusion/src/reader/runtime/liquid_predicate.rs:12-168, plus AND groups), the lowering of
every leaf kind, the argument checks Python makes before the call, and a numpy restatement of the disjunct merge k_sel_or
performs, checked against brute force on odd-sized batches with dirty tails and padding."""
import datetime as dt

import numpy as np
import pyarrow as pa
import pytest

from liquid_cache_b200 import (BinaryExpr, CastExpr, Column, InListExpr, LikeExpr, LiquidExpr, Literal, ScalarFunctionExpr,
                               split_disjunction)
from liquid_cache_b200 import _native as N
from liquid_cache_b200.cache import or_terms, pack_or_terms


def eq(col, v, idx=0):
    return BinaryExpr(Column(col, idx), "=", Literal(v))


def names(parts):
    return [[n for n, _leaf in d] for d in parts]


# ---- split_disjunction ----
def test_reference_three_columns():
    """test_extract_multi_column_or_valid_three_columns: (a = 1 OR b = 2) OR c = 3."""
    expr = BinaryExpr(BinaryExpr(eq("a", 1), "OR", eq("b", 2, 1)), "OR", eq("c", 3, 2))
    parts = split_disjunction(expr)
    assert parts is not None and len(parts) == 3
    assert sorted(n for d in names(parts) for n in d) == ["a", "b", "c"]
    assert all(len(d) == 1 for d in parts)


def test_reference_refusals():
    """test_extract_multi_column_or_invalid_expression: a + b = 5; a single leaf; a = 1 OR (b + c)."""
    assert split_disjunction(BinaryExpr(BinaryExpr(Column("a"), "+", Column("b", 1)), "=", Literal(5))) is None
    assert split_disjunction(eq("a", 1)) is None
    assert split_disjunction(BinaryExpr(eq("a", 1), "OR", BinaryExpr(Column("b", 1), "+", Column("c", 2)))) is None


def test_leaf_kinds():
    like = LikeExpr(False, False, Column("url"), Literal("%google%"))
    like_op = BinaryExpr(Column("ref"), "NotLikeMatch", Literal("%x%"))
    in_list = InListExpr(Column("t"), (Literal(-1), Literal(6)))
    cast = BinaryExpr(CastExpr(CastExpr(Column("EventDate"), pa.int32()), pa.date32()), ">=", Literal(dt.date(2013, 7, 1)))
    expr = BinaryExpr(BinaryExpr(like, "OR", like_op), "OR", BinaryExpr(in_list, "OR", cast))
    parts = split_disjunction(expr)
    assert names(parts) == [["url"], ["ref"], ["t"], ["EventDate"]]
    assert [d[0][1] for d in parts] == [like, like_op, in_list, cast]


def test_dnf_groups():
    q19 = BinaryExpr(BinaryExpr(BinaryExpr(Column("q"), ">=", Literal(1)), "AND", BinaryExpr(Column("q"), "<=", Literal(11))),
                     "OR", BinaryExpr(BinaryExpr(eq("brand", "B#12"), "AND", BinaryExpr(Column("q"), ">=", Literal(10))),
                                      "AND", BinaryExpr(Column("q"), "<=", Literal(20))))
    assert names(split_disjunction(q19)) == [["q", "q"], ["brand", "q", "q"]]
    three = BinaryExpr(BinaryExpr(eq("a", 1), "OR", BinaryExpr(eq("b", 2), "AND", eq("c", 3))), "OR", eq("d", 4))
    assert names(split_disjunction(three)) == [["a"], ["b", "c"], ["d"]]


def test_refused_trees():
    a, b, c = eq("a", 1), eq("b", 2), eq("c", 3)
    assert split_disjunction(BinaryExpr(a, "AND", b)) is None                                 # a conjunction, not an OR
    assert split_disjunction(BinaryExpr(BinaryExpr(a, "OR", b), "AND", c)) is None            # AND over OR is not distributed
    assert split_disjunction(BinaryExpr(a, "OR", BinaryExpr(BinaryExpr(b, "OR", c), "AND", a))) is None  # OR nested in an AND
    assert split_disjunction(BinaryExpr(a, "OR", BinaryExpr(Column("b"), "=", Column("c")))) is None     # column vs column
    assert split_disjunction(BinaryExpr(a, "OR", Literal(True))) is None                                 # a bare literal
    ts = BinaryExpr(ScalarFunctionExpr("to_timestamp_seconds", (Column("t"),)), ">", Literal(5))
    assert split_disjunction(BinaryExpr(a, "OR", ts)) is None                                            # not a cast chain
    assert split_disjunction(BinaryExpr(a, "OR", LikeExpr(False, False, Column("s"), Column("p")))) is None  # pattern not literal
    assert split_disjunction(BinaryExpr(a, "XOR", b)) is None


# ---- lowering and argument checks ----
def test_or_terms_lower_every_leaf_kind():
    h = np.arange(3, dtype=np.uint64)
    leaves = [
        (BinaryExpr(Column("i"), "<", Literal(-5)), pa.int32(), N.OP_LT, N.LIT_I64),
        (BinaryExpr(Column("u"), ">=", Literal(2**63 + 1)), pa.uint64(), N.OP_GE, N.LIT_U64),
        (BinaryExpr(Column("f"), "!=", Literal(0.5)), pa.float64(), N.OP_NE, N.LIT_F64),
        (BinaryExpr(Column("d"), "=", Literal(12)), pa.decimal128(18, 2), N.OP_EQ, N.LIT_I128),
        (BinaryExpr(Column("s"), "=", Literal("MAIL")), pa.string(), N.OP_EQ, N.LIT_BYTES),
        (LikeExpr(False, False, Column("s"), Literal("%google%")), pa.string_view(), N.OP_LIKE, N.LIT_BYTES),
        (LikeExpr(True, False, Column("s"), Literal(b"%x%")), pa.binary(), N.OP_NOT_LIKE, N.LIT_BYTES),
        (InListExpr(Column("i"), (Literal(-1), Literal(6))), pa.int16(), N.OP_IN, N.LIT_I64),
        (InListExpr(Column("s"), (Literal("a"), Literal("bc")), True), pa.dictionary(pa.uint16(), pa.string()), N.OP_NOT_IN, N.LIT_BYTES),
        (Literal(True), pa.string(), N.OP_CONST_TRUE, None),
    ]
    disjuncts = [[(h, LiquidExpr.new_unchecked(e), t)] for e, t, _op, _k in leaves[:4]] + \
                [[(h, LiquidExpr.new_unchecked(e), t) for e, t, _op, _k in leaves[4:]]]
    handles, preds, group = or_terms(disjuncts)
    assert group == [0, 1, 2, 3, 4, 4, 4, 4, 4, 4]
    assert all(x is h for x in handles)
    for p, (_e, _t, op, kind) in zip(preds, leaves):
        assert p.op == op
        if kind is not None:
            assert p.lit_kind == kind
    assert preds[7].lit_len == 2 and preds[3].lit_u64 == 1200  # 12 at scale 2
    with pytest.raises(N.UnsupportedExpr):  # IN on a float column: refused before the call, as Scan.filter refuses it
        or_terms([[(h, LiquidExpr.new_unchecked(InListExpr(Column("f"), (Literal(1.0),))), pa.float64())], [(h, leaves[0][0], pa.int32())]])
    with pytest.raises(ValueError):
        or_terms([])
    with pytest.raises(ValueError):
        or_terms([[(h, LiquidExpr.new_unchecked(leaves[0][0]), pa.int32())], []])


def test_pack_or_terms_checks_before_the_call():
    h = np.arange(4, dtype=np.uint64)
    p = LiquidExpr.new_unchecked(eq("a", 1)).to_native(pa.int32())
    h_ptrs, keep, p_arr, g_arr = pack_or_terms([h, h], [p, p], [0, 0], 4)
    assert len(h_ptrs) == 2 and len(p_arr) == 2 and list(g_arr) == [0, 0] and p_arr[1].op == N.OP_EQ
    assert h_ptrs[0] == keep[0].ctypes.data
    assert pack_or_terms([h], [p], None, 4)[3] is None
    bad = [
        ([], [], None),                 # no terms
        ([h], [p, p], None),            # a handle list missing
        ([h, h[:3]], [p, p], None),     # row counts: 3 handles for 4 batches
        ([h, h], [p, p], [1, 1]),       # group does not start at 0
        ([h, h], [p, p], [0, 2]),       # a gap
        ([h, h, h], [p, p, p], [0, 1, 0]),  # decreasing
        ([h, h], [p, p], [0]),          # one group index for two terms
    ]
    for hs, ps, g in bad:
        with pytest.raises(ValueError):
            pack_or_terms(hs, ps, g, 4)


# ---- the merge step, restated ----
def _layout(rows):
    words = [((r + 31) // 32 + 3) // 4 * 4 for r in rows]
    return np.concatenate([[0], np.cumsum(words)[:-1]]).astype(np.int64), int(sum(words))


def _valid_words(rows, word_off, total):
    v = np.zeros(total, dtype=np.uint32)
    for r, o in zip(rows, word_off):
        v[o:o + r // 32] = 0xFFFFFFFF
        if r % 32:
            v[o + r // 32] = (1 << (r % 32)) - 1
    return v


def sel_or_step(sel, sel_all, term, acc, rows, word_off, first, last):
    """k_sel_or over the whole layout. Returns (sel, term, acc, counts)."""
    valid = _valid_words(rows, word_off, len(term))
    u = ((term if first else acc | term) & valid).astype(np.uint32)
    if last:
        counts = [int(np.unpackbits(u[o:o + ((r + 31) // 32 + 3) // 4 * 4].view(np.uint8)).sum()) for r, o in zip(rows, word_off)]
        return u, term, acc, counts
    s = valid if sel_all else sel
    return sel, (s & ~u & valid).astype(np.uint32), u, None


def _pack(bools, rows, word_off, total, garbage=None):
    w = np.zeros(total, dtype=np.uint32) if garbage is None else garbage.copy()
    for b, (r, o) in enumerate(zip(rows, word_off)):
        n = (r + 31) // 32
        packed = np.packbits(np.concatenate([bools[b], np.zeros(n * 32 - r, dtype=bool)]), bitorder="little").view(np.uint32)
        if garbage is None:
            w[o:o + n] = packed
        else:  # the bits past the row count keep whatever was there, as a refine kernel may leave them
            tail = np.zeros(n, dtype=np.uint32)
            if r % 32:
                tail[-1] = ~np.uint32((1 << (r % 32)) - 1)
            w[o:o + n] = packed | (garbage[o:o + n] & tail)
    return w


@pytest.mark.parametrize("seed", range(6))
def test_merge_restatement_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    rows = [8192, 8191, 1000, 33, 1, 31, 32, 95][: 3 + seed]
    word_off, total = _layout(rows)
    n_disjuncts = int(rng.integers(1, 5))
    terms = [[[rng.random(r) < rng.choice([0.0, 0.3, 0.7, 1.0]) for r in rows] for _ in range(int(rng.integers(1, 4)))]
             for _ in range(n_disjuncts)]
    sel_all = seed % 2 == 0
    start = [np.ones(r, dtype=bool) for r in rows] if sel_all else [rng.random(r) < 0.6 for r in rows]
    sel = np.zeros(total, dtype=np.uint32) if sel_all else _pack(start, rows, word_off, total)
    term = np.zeros(total, dtype=np.uint32)
    acc = rng.integers(0, 2**32, size=total, dtype=np.uint64).astype(np.uint32)  # never read before it is written
    counts = None
    for d, d_terms in enumerate(terms):
        if d == 0:
            term = sel.copy() if not sel_all else None
        for k, mask in enumerate(d_terms):
            # refine_batch: term &= mask (all rows on the very first term when the selection is every row); the words past
            # each batch's rows and its padding are left dirty on purpose
            garbage = rng.integers(0, 2**32, size=total, dtype=np.uint64).astype(np.uint32)
            if term is None:
                term = _pack(mask, rows, word_off, total, garbage)
            else:
                cur = [np.unpackbits(term[o:o + (r + 31) // 32].view(np.uint8), bitorder="little")[:r].astype(bool)
                       for r, o in zip(rows, word_off)]
                term = _pack([c & m for c, m in zip(cur, mask)], rows, word_off, total, garbage)
        sel, term, acc, counts = sel_or_step(sel, sel_all, term, acc, rows, word_off, d == 0, d + 1 == n_disjuncts)
    for b, (r, o) in enumerate(zip(rows, word_off)):
        want = np.zeros(r, dtype=bool)
        for d_terms in terms:
            m = np.ones(r, dtype=bool)
            for mask in d_terms:
                m &= mask[b]
            want |= m
        want &= start[b]
        padded = ((r + 31) // 32 + 3) // 4 * 4
        got_bits = np.unpackbits(sel[o:o + padded].view(np.uint8), bitorder="little")
        assert np.array_equal(got_bits[:r].astype(bool), want), b
        assert not got_bits[r:].any(), f"batch {b}: bits past the row count or in the padding"
        assert counts[b] == int(want.sum())
