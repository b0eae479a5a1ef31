"""GPU parity at BASELINE.json's full sizes, through properties that do not need a second full-size implementation.

The exact per-entry answers come from pyarrow / numpy applied to every batch WHILE it is generated (streaming, one
8192-row batch at a time), so nothing of the 100 M rows is ever kept on the host but a few counters per entry and the
handful of matching rows. Checked on the whole column:
  * every entry's survivor count under the scan pipeline = the Arrow answer for that batch (configs[1], [2], [3])
  * LIKE and NOT LIKE partition the rows of every entry (no nulls in the synthetic URL column)
  * applying a conjunct twice changes nothing (idempotence of selection := selection & valid & cmp)
  * conjunct order does not matter (range AND equality = equality AND range)
  * get-with-selection of the survivors = the Arrow filter of the same rows, bit for bit
  * encode -> decode round trip of sampled entries (insert, then get of every row) and a checksum of checksums over
    the whole integer column (sum of the decoded values of all survivors, wrapping, = numpy's)
LC_SCALE_ROWS shrinks the workload for quick runs (default: the 100 M rows bench.py uses; nearly all of a
test's time goes to generating the synthetic input).
"""
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = pytest.mark.gpu

ROWS = int(os.environ.get("LC_SCALE_ROWS", "100000000"))
ROWS_PER_ENTRY = 8192


@pytest.fixture()
def big_cache():
    """A cache of its own: the column is released when the test ends."""
    from liquid_cache_b200 import LiquidCacheBuilder

    c = LiquidCacheBuilder.new().build()
    yield c
    c.close()


def test_url_like_full_size(big_cache):
    import bench
    from liquid_cache_b200 import CacheExpression, Column, LikeExpr, LiquidExpr, Literal, parquet_array_id

    cache = big_cache
    n_entries = max(1, ROWS // ROWS_PER_ENTRY)
    want_counts = np.zeros(n_entries, dtype=np.uint64)
    want_rows, ids, sample = [], [], {}
    for i, arr in bench.generate_entries(0, n_entries, min(32, os.cpu_count() or 8)):
        eid = parquet_array_id(0, i // 32, 13, i % 32)
        cache.insert(eid, arr).with_squeeze_hint(CacheExpression.SubstringSearch).run()
        ids.append(int(eid))
        hit = pc.match_substring(arr, "google")
        k = pc.sum(hit).as_py() or 0
        want_counts[i] = k
        if k:
            want_rows.append(arr.filter(hit))
        if i % max(1, n_entries // 8) == 0:
            sample[i] = arr
    handles = cache.handles(ids)
    rows = np.full(n_entries, ROWS_PER_ENTRY, dtype=np.uint64)

    def native(negated):
        e = LiquidExpr.try_new(LikeExpr(negated, False, Column("URL", 0), Literal("%google%")), pa.string(), CacheExpression.SubstringSearch)
        assert e is not None
        return e.to_native(pa.string())

    with cache.scan(rows) as scan:
        scan.filter_native(handles, native(False))
        counts, total = scan.counts()
        assert np.array_equal(counts, want_counts), f"{int((counts != want_counts).sum())} entries disagree with Arrow"
        assert total == int(want_counts.sum())
        got = scan.read(handles) if total else None
        scan.filter_native(handles, native(False))  # idempotence
        counts2, total2 = scan.counts()
        assert np.array_equal(counts2, counts) and total2 == total
        if total:
            assert scan.read(handles).equals(got)
            assert got.equals(pa.concat_arrays(want_rows)), "get-with-selection differs from the Arrow filter"
        scan.reset()
        scan.filter_native(handles, native(True))  # NOT LIKE: the complement (the column has no nulls)
        ncounts, ntotal = scan.counts()
        assert np.array_equal(ncounts + counts, rows) and ntotal + total == n_entries * ROWS_PER_ENTRY
    for i, arr in sample.items():  # encode -> decode round trip
        assert cache.get(ids[i]).read().equals(arr), f"entry {i} does not round-trip"


def _int_column_full_size(cache, column, seed, col_id, conjuncts, arrow_type):
    """Insert the column, run the conjuncts in both orders, return nothing; asserts inside."""
    import synth
    from liquid_cache_b200 import BinaryExpr, Column, LiquidExpr, Literal, parquet_array_id

    n_entries = max(1, ROWS // ROWS_PER_ENTRY)
    want_counts = np.zeros(n_entries, dtype=np.uint64)
    want_sum = 0
    ids, want_rows, sample = [], [], {}
    group = 1024
    ops = {">=": pc.greater_equal, "<": pc.less, "=": pc.equal}
    plain = pa.int32() if arrow_type == pa.date32() else pa.int64()
    for g0 in range(0, n_entries, group):
        idx = range(g0, min(n_entries, g0 + group))
        batches = [synth.int_entry(column, i, seed=seed) for i in idx]
        eids = [parquet_array_id(2, i // 32, col_id, i % 32) for i in idx]
        cache.insert_many(eids, batches)
        ids.extend(int(e) for e in eids)
        big = pa.concat_arrays(batches)  # the Arrow answer for the whole group in one vectorised pass
        m = None
        for op, lit in conjuncts:
            c = ops[op](big, pa.scalar(lit, arrow_type))
            m = c if m is None else pc.and_(m, c)
        want_counts[g0:g0 + len(batches)] = np.asarray(m.to_numpy(zero_copy_only=False)).reshape(-1, ROWS_PER_ENTRY).sum(axis=1)
        f = big.filter(m)
        if len(f):
            want_rows.append(f)
            want_sum = (want_sum + int(np.asarray(f.cast(plain)).astype(np.int64).sum())) & (2**64 - 1)
        for i, arr in zip(idx, batches):
            if i % max(1, n_entries // 8) == 0:
                sample[i] = arr
    handles = cache.handles(ids)
    rows = np.full(n_entries, ROWS_PER_ENTRY, dtype=np.uint64)

    def native(op, lit):
        return LiquidExpr.new_unchecked(BinaryExpr(Column(column, 0), op, Literal(lit))).to_native(arrow_type)

    with cache.scan(rows) as scan:
        for op, lit in conjuncts:
            scan.filter_native(handles, native(op, lit))
        counts, total = scan.counts()
        assert np.array_equal(counts, want_counts), f"{int((counts != want_counts).sum())} entries disagree with Arrow"
        got = scan.read(handles)
        want = pa.concat_arrays(want_rows) if want_rows else pa.array([], arrow_type)
        assert got.equals(want), "get-with-selection differs from the Arrow filter"
        got_np = np.asarray(got.cast(plain)).astype(np.int64)
        assert (int(got_np.sum()) & (2**64 - 1)) == want_sum  # checksum of checksums
        scan.filter_native(handles, native(*conjuncts[0]))  # idempotence
        counts2, _ = scan.counts()
        assert np.array_equal(counts2, counts)
        scan.reset()
        for op, lit in reversed(conjuncts):  # order independence
            scan.filter_native(handles, native(op, lit))
        counts3, total3 = scan.counts()
        assert np.array_equal(counts3, counts) and total3 == total
    for i, arr in sample.items():
        assert cache.get(ids[i]).read().equals(arr), f"entry {i} does not round-trip"


def test_event_time_range_full_size(big_cache):
    """configs[2] shape: EventTime (Int64, W = 17) range of two conjuncts."""
    import synth

    lo = 1373832014 + 20000
    _int_column_full_size(big_cache, "EventTime", synth.SEED_INT, 4, [(">=", lo), ("<", lo + 8640)], pa.int64())


def test_user_id_equality_full_size(big_cache):
    """configs[2] shape: UserID (Int64, W = 64) equality on a value that occurs."""
    import synth

    uid = int(synth.int_entry("UserID", 0, seed=synth.SEED_INT)[17].as_py())
    _int_column_full_size(big_cache, "UserID", synth.SEED_INT, 9, [("=", uid)], pa.int64())


def test_shipdate_range_full_size(big_cache):
    """configs[3] shape: l_shipdate (Date32, W = 12), q6's one-year range; one GPU's eighth of SF100 by default."""
    import datetime as dt

    import synth

    global ROWS
    saved = ROWS
    try:
        ROWS = min(ROWS, 600_037_902 // 8)
        _int_column_full_size(big_cache, "l_shipdate", synth.SEED_TPCH, 10,
                              [(">=", dt.date(1994, 1, 1)), ("<", dt.date(1995, 1, 1))], pa.date32())
    finally:
        ROWS = saved
