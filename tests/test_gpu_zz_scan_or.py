"""lc_scan_filter_or: an OR of AND groups of single-column predicates as one conjunct of the device scan. Every case is checked
per batch against pyarrow on the decoded columns: selection & OR_d AND_t fill_null(mask_t, False), with the counts. The
reference evaluates the pure-OR shape with try_eval_predicate per leaf and or_kleene (src/datafusion/src/cache/mod.rs:
111-150); a null leaf is false once the reader turns null into false, which is what the scan computes per term."""
import ctypes as C
import decimal
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from liquid_cache_b200 import (BinaryExpr, CacheExpression, Column, InListExpr, LikeExpr, LiquidExpr, Literal,
                               split_disjunction)
from liquid_cache_b200 import _native as N
from oracle import liquid_oracle as O
from tests.golden_cases import MULTI_COLUMN_OR_CASES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = [8192, 8191, 1000, 33, 8192, 5000]
CMP = {"=": pc.equal, "!=": pc.not_equal, "<": pc.less, "<=": pc.less_equal, ">": pc.greater, ">=": pc.greater_equal}
POOL = ["", "a", "MAIL", "SHIP", "AIR", "AIR REG", "TRUCK", "http://www.google.com/search?q=1", "http://yandex.ru/page/2",
        "http://example.org/page/22", "https://mail.google.com/inbox/" + "z" * 40, "x" * 300, "x" * 300 + "y", "SM CASE", "LG PACK"]


class Col:
    """One column of the scan: a batch per entry of ROWS (or `rows`), its device entries and the original arrays."""

    def __init__(self, cache, arrays, hint=None):
        self.arrays = arrays
        self.type = arrays[0].type
        self.g = [cache.transcode(a, hint=hint) for a in arrays]
        self.h = np.array([g.handle for g in self.g], dtype=np.uint64)


def _plain(a):
    """The decoded column as Arrow compares it: dictionaries decoded, byte views and binaries as Utf8 (ASCII data)."""
    if pa.types.is_dictionary(a.type):
        a = a.cast(a.type.value_type)
    if pa.types.is_binary(a.type) or pa.types.is_binary_view(a.type) or pa.types.is_string_view(a.type):
        a = a.cast(pa.string())
    return a


def arrow_leaf(arr, op, lit):
    a = _plain(arr)
    if op in ("like", "not like"):
        m = pc.match_like(a, lit)
        m = pc.invert(m) if op == "not like" else m
    elif op in ("in", "not in"):
        m = pc.is_in(a, value_set=pa.array(list(lit), a.type))
        m = pc.invert(m) if op == "not in" else m
        m = pc.if_else(pc.is_null(a), pa.scalar(None, pa.bool_()), m)
    else:
        m = CMP[op](a, pa.scalar(lit, a.type))
    return np.asarray(m.fill_null(False).to_numpy(zero_copy_only=False), dtype=bool)


def leaf_expr(op, lit, binary=False):
    enc = (lambda v: v.encode()) if binary else (lambda v: v)
    col = Column("c", 0)
    if op in ("like", "not like"):
        return LiquidExpr.new_unchecked(LikeExpr(op == "not like", False, col, Literal(enc(lit))))
    if op in ("in", "not in"):
        return LiquidExpr.new_unchecked(InListExpr(col, tuple(Literal(enc(v)) for v in lit), op == "not in"))
    return LiquidExpr.new_unchecked(BinaryExpr(col, op, Literal(enc(lit))))


def is_binary(col):
    t = col.type.value_type if pa.types.is_dictionary(col.type) else col.type
    return pa.types.is_binary(t) or pa.types.is_binary_view(t)


def expected(cols_terms, start):
    """start[b] & OR_d AND_t leaf_t, per batch. cols_terms = [[(col, op, lit), ...], ...]."""
    out = []
    for b, s in enumerate(start):
        acc = np.zeros(len(s), dtype=bool)
        for d in cols_terms:
            m = np.ones(len(s), dtype=bool)
            for col, op, lit in d:
                m &= arrow_leaf(col.arrays[b], op, lit)
            acc |= m
        out.append(s & acc)
    return out


def run_or(sc, cols_terms):
    sc.filter_or([[(col.h, leaf_expr(op, lit, is_binary(col)), col.type) for col, op, lit in d] for d in cols_terms])


def meaningful_words(sc, rows):
    """The selection words that carry rows (store_selections zeroes the bits past each batch's rows; the padding words up to
    the batch's 4-word boundary carry nothing and are left out)."""
    words = sc.store_selections()
    offs, _total = sc.selection_layout()
    return np.concatenate([words[int(o):int(o) + (r + 31) // 32] for o, r in zip(offs, rows)])


def check(sc, want, what):
    counts, total = sc.counts()
    assert [int(c) for c in counts] == [int(w.sum()) for w in want], what
    assert total == sum(int(w.sum()) for w in want), what
    for b, w in enumerate(want):
        got = np.asarray(sc.selection(b).to_numpy(zero_copy_only=False), dtype=bool)
        assert np.array_equal(got, w), f"{what}: batch {b}, {np.flatnonzero(got != w)[:8]}"


# ---- columns ----
def _ints(rng, typ, rows, lo, hi, null_p=0.1):
    out = []
    for r in rows:
        vals = rng.integers(lo, hi, size=r, endpoint=True, dtype=np.int64 if lo < 0 else np.uint64)
        out.append(pa.array(vals, type=pa.int64() if lo < 0 else pa.uint64(), mask=rng.random(r) < null_p).cast(typ))
    return out


def _strings(rng, rows, kind="utf8", null_p=0.1):
    out = []
    for r in rows:
        if kind == "dict":
            idx = pa.array(rng.integers(0, len(POOL), size=r), pa.uint16(), mask=rng.random(r) < null_p)
            out.append(pa.DictionaryArray.from_arrays(idx, pa.array(POOL)))
            continue
        a = pa.array([POOL[i] for i in rng.integers(0, len(POOL), size=r)], pa.string(), mask=rng.random(r) < null_p)
        out.append(a.cast({"utf8": pa.string(), "binary": pa.binary(), "utf8_view": pa.string_view()}[kind]))
    return out


INT_KINDS = [(pa.int8(), -128, 127), (pa.uint8(), 0, 255), (pa.int16(), -3000, 3000), (pa.uint16(), 0, 65535),
             (pa.int32(), -(2**31), 2**31 - 1), (pa.uint32(), 0, 2**32 - 1), (pa.int64(), -(2**62), 2**62), (pa.uint64(), 0, 2**64 - 1)]


def make_columns(cache, rng, rows):
    cols = {}
    for typ, lo, hi in INT_KINDS:
        narrow_lo = max(lo, -200)
        cols[str(typ)] = Col(cache, _ints(rng, typ, rows, narrow_lo, min(hi, narrow_lo + 400)))
    cols["int64_wide"] = Col(cache, _ints(rng, pa.int64(), rows, -(2**50), 2**50))
    cols["date32"] = Col(cache, [a.cast(pa.date32()) for a in _ints(rng, pa.int32(), rows, 15000, 15300)])
    cols["timestamp"] = Col(cache, [a.cast(pa.timestamp("us")) for a in _ints(rng, pa.int64(), rows, 10**12, 10**12 + 10**6)])
    cols["float64"] = Col(cache, [pa.array(np.round(rng.random(r) * 100, 2), mask=rng.random(r) < 0.1) for r in rows])
    cols["decimal_u64"] = Col(cache, [a.cast(pa.decimal128(22, 2)) for a in _ints(rng, pa.int64(), rows, 0, 5000)])
    cols["decimal_fixed"] = Col(cache, [pa.array([None if v is None else decimal.Decimal(v).scaleb(-2) for v in a.to_pylist()],
                                                 pa.decimal128(38, 2)) for a in _ints(rng, pa.int64(), rows, -(2**62), 2**62)])
    for kind in ("utf8", "binary", "utf8_view", "dict"):
        cols[kind] = Col(cache, _strings(rng, rows, kind), hint=CacheExpression.SubstringSearch)
    return cols


def random_leaf(rng, name, col):
    """(op, literal) on `col` with a literal drawn from its data (a selective but non-empty predicate, mostly)."""
    plain = [a.cast(pa.int64()) if pa.types.is_timestamp(a.type) else _plain(a) for a in col.arrays[:2]]  # timestamps: ticks
    vals = [v for a in plain for v in a.to_pylist() if v is not None]
    pick = lambda: vals[int(rng.integers(0, len(vals)))]  # noqa: E731
    if name in ("utf8", "binary", "utf8_view", "dict"):
        kind = int(rng.integers(0, 6))
        if kind == 0:
            return ("like", "%google%") if rng.random() < 0.5 else ("like", "%mail.google.com/inbox/" + "z" * 20 + "%")
        if kind == 1:
            return ("not like", "%example%")
        if kind == 2:
            return ("in", [pick(), pick(), "absent"])
        if kind == 3:
            return ("not in", [pick(), "x" * 300])
        return (["=", "!=", "<", ">="][int(rng.integers(0, 4))], pick())
    if name in ("float64", "decimal_u64", "decimal_fixed"):
        return (list(CMP)[int(rng.integers(0, 6))], pick())
    if rng.random() < 0.3:
        return ("in" if rng.random() < 0.5 else "not in", [pick() for _ in range(int(rng.integers(1, 5)))])
    return (list(CMP)[int(rng.integers(0, 6))], pick())


# ---- tests ----
def test_reference_known_answers(cache):
    """The reference's three multi-column OR cases (evaluate_selection_with_predicate), through the scan."""
    types = {"int32": pa.int32(), "string_view": pa.string_view()}
    for case, (cols, conjuncts, want_rows) in enumerate(MULTI_COLUMN_OR_CASES):
        n = len(cols[0][1])
        arrays = [pa.array(vals, types[t]) for t, vals in cols]
        cs = [Col(cache, [a]) for a in arrays]
        restated = O.evaluate_multi_column_or([(O.transcode(a), op, lit) for a, (op, lit) in zip(arrays, conjuncts)],
                                              pa.array([True] * n))
        full = [bool(x) for x in restated.fill_null(False).to_pylist()]
        assert full == [i in want_rows for i in range(n)], case
        for sel in (None, [i % 2 == 1 for i in range(n)]):
            with cache.scan([n]) as sc:
                if sel is not None:
                    sc.set_selection(0, pa.array(sel))
                sc.filter_or([[(c.h, LiquidExpr.new_unchecked(BinaryExpr(Column(f"c{i}", i), op, Literal(lit))), c.type)]
                              for i, (c, (op, lit)) in enumerate(zip(cs, conjuncts))])
                got = sc.selection(0).to_pylist()
                counts, total = sc.counts()
            want = [f and (sel is None or sel[i]) for i, f in enumerate(full)]
            assert got == want and total == sum(want), (case, sel is not None)


@pytest.mark.parametrize("start", ["all", "seeded", "filtered"])
def test_random_terms_over_every_type(cache, start):
    rng = np.random.default_rng({"all": 1, "seeded": 2, "filtered": 3}[start])
    cols = make_columns(cache, rng, ROWS)
    names = list(cols)
    for round_ in range(40):
        n_terms = int(rng.integers(2, 6))
        terms = []
        for _ in range(n_terms):
            name = names[int(rng.integers(0, len(names)))]
            op, lit = random_leaf(rng, name, cols[name])
            terms.append((cols[name], op, lit, name))
        cuts = sorted(set(int(x) for x in rng.integers(1, n_terms, size=int(rng.integers(0, n_terms)))))
        bounds = [0] + cuts + [n_terms]
        dnf = [[t[:3] for t in terms[a:b]] for a, b in zip(bounds, bounds[1:])]
        with cache.scan(ROWS) as sc:
            base = [np.ones(r, dtype=bool) for r in ROWS]
            if start == "seeded":
                base = [rng.random(r) < 0.6 for r in ROWS]
                for b, s in enumerate(base):
                    sc.set_selection(b, pa.array(s))
            elif start == "filtered":
                c = cols["int32"]
                sc.filter(c.h, leaf_expr(">", -120), c.type)
                base = [arrow_leaf(a, ">", -120) for a in c.arrays]
            run_or(sc, dnf)
            check(sc, expected(dnf, base), f"{start} round {round_}: {[[(t[3], t[1], str(t[2])[:40]) for t in terms]]} cuts={cuts}")


def test_dnf_groups_edge_cases(cache):
    rng = np.random.default_rng(7)
    a = Col(cache, _ints(rng, pa.int32(), ROWS, 0, 50))
    s = Col(cache, _strings(rng, ROWS), hint=CacheExpression.SubstringSearch)
    cases = [
        [[(a, ">=", 10), (a, "<=", 20)], [(s, "=", "MAIL")]],             # q19 shape: the same column twice in one group
        [[(a, "<", 0)], [(s, "like", "%google%")]],                      # a disjunct that selects nothing
        [[(a, ">=", 0)], [(s, "=", "SHIP")]],                            # one that selects every valid row
        [[(s, "like", "%google%"), (a, "!=", 3)], [(a, "in", [1, 2, 3]), (s, "not like", "%x%")], [(a, "=", 49)]],
        [[(a, "<", 0)], [(a, ">", 100)]],                                # nothing at all
        [[(s, "!=", "nope"), (a, ">=", 0), (a, "<=", 50)]],              # one disjunct: an AND group
    ]
    for i, dnf in enumerate(cases):
        for seeded in (False, True):
            with cache.scan(ROWS) as sc:
                base = [np.ones(r, dtype=bool) for r in ROWS]
                if seeded:
                    base = [np.arange(r) % 3 != 0 for r in ROWS]
                    for b, sel in enumerate(base):
                        sc.set_selection(b, pa.array(sel))
                run_or(sc, dnf)
                check(sc, expected(dnf, base), f"case {i} seeded={seeded}")
                run_or(sc, dnf)  # again, on the result: idempotent
                check(sc, expected(dnf, base), f"case {i} seeded={seeded}, twice")


def test_one_term_matches_scan_filter_bit_for_bit(cache):
    rng = np.random.default_rng(9)
    cols = make_columns(cache, rng, ROWS)
    for name in ("int32", "int64_wide", "float64", "utf8", "dict", "decimal_fixed"):
        col = cols[name]
        op, lit = random_leaf(rng, name, col)
        for seeded in (False, True):
            with cache.scan(ROWS) as want_sc, cache.scan(ROWS) as got_sc:
                if seeded:
                    for b, r in enumerate(ROWS):
                        sel = pa.array(np.arange(r) % 5 != 1)
                        want_sc.set_selection(b, sel)
                        got_sc.set_selection(b, sel)
                want_sc.filter(col.h, leaf_expr(op, lit, is_binary(col)), col.type)
                got_sc.filter_or([[(col.h, leaf_expr(op, lit, is_binary(col)), col.type)]])
                assert np.array_equal(meaningful_words(got_sc, ROWS), meaningful_words(want_sc, ROWS)), (name, op)
                wc, wt = want_sc.counts()
                gc, gt = got_sc.counts()
                assert np.array_equal(gc, wc) and gt == wt, (name, op)


def test_squeezed_entries_in_a_term(cache):
    rng = np.random.default_rng(11)
    arrays = [pa.array(rng.integers(-(2**40), -(2**40) + (1 << 20), size=r), pa.int64()) for r in ROWS]
    fulls, mixed, keep = [], [], []
    for b, arr in enumerate(arrays):
        full = cache.transcode(arr)
        entry = full
        form = ("full", "clamp", "quantize")[b % 3]
        if form != "full":
            class Io:
                def read(self, rng_):
                    return self.bytes[rng_[0]:rng_[1]]
            io = Io()
            entry, image = full.squeeze(io, CacheExpression.PredicateColumn, form)
            io.bytes = image
            keep.append(io)
        fulls.append(full.handle)
        mixed.append(entry.handle)
        keep.append((full, entry))
    h_full, h_mixed = np.array(fulls, dtype=np.uint64), np.array(mixed, dtype=np.uint64)
    s = Col(cache, _strings(rng, ROWS), hint=CacheExpression.SubstringSearch)
    vals = np.concatenate([a.to_numpy() for a in arrays])
    lo, hi, present = int(np.quantile(vals, 0.2)), int(np.quantile(vals, 0.7)), int(vals[17])
    for ops in ([(">=", lo), ("<", hi)], [("=", present)], [("<", int(vals.min()))]):
        for seeded in (False, True):
            with cache.scan(ROWS) as want_sc, cache.scan(ROWS) as got_sc:
                if seeded:
                    for b, r in enumerate(ROWS):
                        sel = pa.array(np.arange(r) % 4 != 2)
                        want_sc.set_selection(b, sel)
                        got_sc.set_selection(b, sel)
                for sc, h in ((want_sc, h_full), (got_sc, h_mixed)):
                    group = [(h, leaf_expr(op, k), pa.int64()) for op, k in ops]
                    sc.filter_or([group, [(s.h, leaf_expr("=", "TRUCK"), s.type)]])
                assert np.array_equal(meaningful_words(got_sc, ROWS), meaningful_words(want_sc, ROWS)), ops
                wc, wt = want_sc.counts()
                gc, gt = got_sc.counts()
                assert np.array_equal(gc, wc) and gt == wt, ops
                base = [np.arange(r) % 4 != 2 if seeded else np.ones(r, dtype=bool) for r in ROWS]
                want = []
                for b, r in enumerate(ROWS):
                    m = np.ones(r, dtype=bool)
                    for op, k in ops:
                        m &= arrow_leaf(arrays[b], op, k)
                    want.append(base[b] & (m | arrow_leaf(s.arrays[b], "=", "TRUCK")))
                check(got_sc, want, f"squeezed {ops} seeded={seeded}")


def test_read_after_or_equals_arrow_filter(cache):
    rng = np.random.default_rng(13)
    a = Col(cache, _ints(rng, pa.int32(), ROWS, 0, 1000, 0.0))
    s = Col(cache, _strings(rng, ROWS, null_p=0.0), hint=CacheExpression.SubstringSearch)
    dnf = [[(s, "like", "%google%")], [(a, "<", 30), (a, ">", 10)]]
    with cache.scan(ROWS) as sc:
        run_or(sc, dnf)
        want = expected(dnf, [np.ones(r, dtype=bool) for r in ROWS])
        want_s = pa.concat_arrays([arr.filter(pa.array(w)) for arr, w in zip(s.arrays, want)])
        want_a = pa.concat_arrays([arr.filter(pa.array(w)) for arr, w in zip(a.arrays, want)])
        for _ in range(2):  # the second read is planned from the first one's sizes
            assert sc.read(s.h).to_pylist() == want_s.to_pylist()
            assert sc.read(a.h).to_pylist() == want_a.to_pylist()


def _in_on_float():
    p = N.Predicate()
    p.op, p.lit_kind, p.lit_len = N.OP_IN, N.LIT_I64, 1
    one = np.array([1], dtype="<i8").tobytes()
    p._keepalive = one
    p.lit_bytes = one
    return p


def test_refusals_leave_the_selection_and_counts_unchanged(cache):
    rng = np.random.default_rng(15)
    a = Col(cache, _ints(rng, pa.int32(), ROWS, 0, 100))
    f = Col(cache, [pa.array(rng.random(r)) for r in ROWS])
    short = Col(cache, _ints(rng, pa.int32(), [r + 1 for r in ROWS], 0, 100))
    good = [leaf_expr("<", 50).to_native(pa.int32()), leaf_expr(">", 90).to_native(pa.int32())]
    with cache.scan(ROWS) as sc:
        sc.filter(a.h, leaf_expr("!=", 7), pa.int32())
        before, before_counts = sc.store_selections().copy(), sc.counts()
        for pos in range(3):  # the float IN term first, in the middle, last
            preds = list(good)
            preds.insert(pos, _in_on_float())
            hs = [a.h, a.h]
            hs.insert(pos, f.h)
            for group in (None, [0, 0, 1]):
                with pytest.raises(N.UnsupportedExpr):
                    sc.filter_or_native(hs, preds, group)
                assert np.array_equal(sc.store_selections(), before), (pos, group)
                c, t = sc.counts()
                assert np.array_equal(c, before_counts[0]) and t == before_counts[1]
        lib = N.lib()
        arr_h = (C.c_void_p * 2)(a.h.ctypes.data, a.h.ctypes.data)
        arr_p = (N.Predicate * 2)(*good)
        bad_calls = [
            lambda: lib.lc_scan_filter_or(sc._scan, 0, arr_h, arr_p, None),                            # no terms
            lambda: lib.lc_scan_filter_or(sc._scan, 2, None, arr_p, None),                             # no handles
            lambda: lib.lc_scan_filter_or(sc._scan, 2, arr_h, None, None),                             # no predicates
            lambda: lib.lc_scan_filter_or(sc._scan, 2, (C.c_void_p * 2)(a.h.ctypes.data, None), arr_p, None),
            lambda: lib.lc_scan_filter_or(sc._scan, 2, arr_h, arr_p, (C.c_uint32 * 2)(1, 1)),          # group not from 0
            lambda: lib.lc_scan_filter_or(sc._scan, 2, arr_h, arr_p, (C.c_uint32 * 2)(0, 2)),          # a gap
            lambda: lib.lc_scan_filter_or(sc._scan, 2, arr_h, arr_p, (C.c_uint32 * 2)(1, 0)),          # decreasing
            lambda: lib.lc_scan_filter_or(sc._scan, 2, (C.c_void_p * 2)(a.h.ctypes.data, short.h.ctypes.data), arr_p, None),
            lambda: lib.lc_scan_filter_or(None, 2, arr_h, arr_p, None),
        ]
        for i, call in enumerate(bad_calls):
            assert call() == N.LC_ERR_INVALID, i
            assert np.array_equal(sc.store_selections(), before), i
            c, t = sc.counts()
            assert np.array_equal(c, before_counts[0]) and t == before_counts[1], i
        with pytest.raises(ValueError):
            sc.filter_or_native([a.h], good, None)  # two predicates, one handle list
        with pytest.raises(ValueError):
            sc.filter_or_native([a.h, a.h], good, [0, 2])


def test_launches_are_the_terms_plus_one_merge_per_disjunct(cache):
    rng = np.random.default_rng(17)
    a = Col(cache, _ints(rng, pa.int32(), ROWS, 0, 1000, 0.0))
    w = Col(cache, _ints(rng, pa.int64(), ROWS, -(2**50), 2**50, 0.0))
    f = Col(cache, [pa.array(rng.random(r)) for r in ROWS])
    s1 = Col(cache, _strings(rng, ROWS), hint=CacheExpression.SubstringSearch)
    s2 = Col(cache, _strings(rng, ROWS, "utf8_view"), hint=CacheExpression.SubstringSearch)
    dnf = [[(s1, "like", "%google%"), (a, "<", 500)], [(f, ">", 0.25), (w, ">", 0)], [(s2, "like", "%mail%")], [(a, "in", [1, 5, 9])]]
    with cache.scan(ROWS) as sc:
        run_or(sc, dnf)  # warms the entry lists and the LIKE step tables
        per_term = 0
        for d in dnf:
            for col, op, lit in d:
                k0 = cache.stats().kernel_launches
                sc.filter(col.h, leaf_expr(op, lit, is_binary(col)), col.type)
                per_term += cache.stats().kernel_launches - k0
        sc.reset()
        st0 = cache.stats()
        run_or(sc, dnf)
        st1 = cache.stats()
        assert st1.kernel_launches - st0.kernel_launches == per_term + len(dnf)
        assert st1.d2h_bytes == st0.d2h_bytes
        sc.counts()
        check(sc, expected(dnf, [np.ones(r, dtype=bool) for r in ROWS]), "cost case")


def test_split_disjunction_feeds_the_scan(cache):
    rng = np.random.default_rng(19)
    a = Col(cache, _ints(rng, pa.int32(), ROWS, 0, 100))
    s = Col(cache, _strings(rng, ROWS), hint=CacheExpression.SubstringSearch)
    cols = {"a": a, "s": s}
    tree = BinaryExpr(BinaryExpr(BinaryExpr(Column("a"), ">=", Literal(10)), "AND", BinaryExpr(Column("a"), "<=", Literal(20))),
                      "OR", LikeExpr(False, False, Column("s"), Literal("%google%")))
    parts = split_disjunction(tree)
    assert [[n for n, _ in d] for d in parts] == [["a", "a"], ["s"]]
    with cache.scan(ROWS) as sc:
        sc.filter_or([[(cols[n].h, LiquidExpr.new_unchecked(leaf), cols[n].type) for n, leaf in d] for d in parts])
        check(sc, expected([[(a, ">=", 10), (a, "<=", 20)], [(s, "like", "%google%")]], [np.ones(r, dtype=bool) for r in ROWS]),
              "split tree")


def test_c_mirror_program():
    lib_dir = os.path.join(ROOT, "liquid_cache_b200", "lib")
    exe = os.path.join(ROOT, "build", "tests", "scan_or_mirror")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    r = subprocess.run(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT}", os.path.join(ROOT, "tests", "cpp", "scan_or_mirror.c"),
                        "-o", exe, f"-L{lib_dir}", "-llc_gpu", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "0 wrong answers" in r.stdout, (r.returncode, r.stdout, r.stderr)
