"""bench.py --workload clickbench_sweep — the scan stage of the 43 ClickBench queries over an HBM-resident `hits`
(BASELINE.json configs[4], SURVEY.md §8d row 5 and its table of per-query scan shapes).

What reaches the cache for a query is (conjuncts in the reader's priority order, projected columns); everything above
that (GROUP BY, ORDER BY, aggregates) is DataFusion's and is not part of this path. Per query the sweep does what
LiquidCacheReader does for every batch of the table (src/datafusion/src/reader/runtime/liquid_cache_reader.rs:297-391),
batched over all entries: every conjunct refines the running selection on the device (lc_scan_filter), one small D2H
returns the survivor counts, and every projected column is read with the final selection (device-resident:
lc_scan_read_device; e2e: lc_scan_read, Arrow arrays on the host). Conjuncts the path does not push down (q40's IN list —
liquid_expr.rs admits no InListExpr) are evaluated the reference's way: get-with-selection, Arrow on the CPU, selection
written back.

Literals: the 24 586-row sample the generator draws from (synth/hits.py) has no CounterID 62 and none of the hash / UserID
constants of the official queries, so those literals are replaced by values that occur in the sample (noted per query as
"literal from sample"); patterns and date ranges are the official ones.
"""
from __future__ import annotations

import datetime as dt
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ROWS_PER_ENTRY = 8192
D = dt.date

# (query, [(column, op, literal)], [projected columns])   — benchmark/clickbench/queries/q0.sql .. q42.sql.
# Conjunct order = row_filter.rs:501-515 (`=` / `<>` first, then LIKE, NOT LIKE, ranges). "@X" = literal taken from the sample.
_JULY = [("EventDate", ">=", D(2013, 7, 1)), ("EventDate", "<=", D(2013, 7, 31))]
QUERIES = [
    (0, [], []),
    (1, [("AdvEngineID", "!=", 0)], []),
    (2, [], ["AdvEngineID", "ResolutionWidth"]),
    (3, [], ["UserID"]),
    (4, [], ["UserID"]),
    (5, [], ["SearchPhrase"]),
    (6, [], ["EventDate"]),
    (7, [("AdvEngineID", "!=", 0)], ["AdvEngineID"]),
    (8, [], ["RegionID", "UserID"]),
    (9, [], ["RegionID", "AdvEngineID", "ResolutionWidth", "UserID"]),
    (10, [("MobilePhoneModel", "!=", "")], ["MobilePhoneModel", "UserID"]),
    (11, [("MobilePhoneModel", "!=", "")], ["MobilePhone", "MobilePhoneModel", "UserID"]),
    (12, [("SearchPhrase", "!=", "")], ["SearchPhrase"]),
    (13, [("SearchPhrase", "!=", "")], ["SearchPhrase", "UserID"]),
    (14, [("SearchPhrase", "!=", "")], ["SearchEngineID", "SearchPhrase"]),
    (15, [], ["UserID"]),
    (16, [], ["UserID", "SearchPhrase"]),
    (17, [], ["UserID", "SearchPhrase"]),
    (18, [], ["UserID", "EventTime", "SearchPhrase"]),
    (19, [("UserID", "=", "@UserID")], ["UserID"]),
    (20, [("URL", "like", "%google%")], []),
    (21, [("SearchPhrase", "!=", ""), ("URL", "like", "%google%")], ["SearchPhrase", "URL"]),
    (22, [("SearchPhrase", "!=", ""), ("Title", "like", "%Google%"), ("URL", "not like", "%.google.%")],
     ["SearchPhrase", "URL", "Title", "UserID"]),
    (23, [("URL", "like", "%google%")], ["EventTime", "URL", "Title", "Referer", "SearchPhrase", "UserID", "WatchID", "CounterID"]),
    (24, [("SearchPhrase", "!=", "")], ["SearchPhrase", "EventTime"]),
    (25, [("SearchPhrase", "!=", "")], ["SearchPhrase"]),
    (26, [("SearchPhrase", "!=", "")], ["SearchPhrase", "EventTime"]),
    (27, [("URL", "!=", "")], ["CounterID", "URL"]),
    (28, [("Referer", "!=", "")], ["Referer"]),
    (29, [], ["ResolutionWidth"]),
    (30, [("SearchPhrase", "!=", "")], ["SearchEngineID", "ClientIP", "IsRefresh", "ResolutionWidth"]),
    (31, [("SearchPhrase", "!=", "")], ["WatchID", "ClientIP", "IsRefresh", "ResolutionWidth"]),
    (32, [], ["WatchID", "ClientIP", "IsRefresh", "ResolutionWidth"]),
    (33, [], ["URL"]),
    (34, [], ["URL"]),
    (35, [], ["ClientIP"]),
    (36, [("CounterID", "=", "@CounterID"), ("DontCountHits", "=", 0), ("IsRefresh", "=", 0), ("URL", "!=", "")] + _JULY, ["URL"]),
    (37, [("CounterID", "=", "@CounterID"), ("DontCountHits", "=", 0), ("IsRefresh", "=", 0), ("Title", "!=", "")] + _JULY, ["Title"]),
    (38, [("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0), ("IsLink", "!=", 0), ("IsDownload", "=", 0)] + _JULY, ["URL"]),
    (39, [("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0)] + _JULY,
     ["TraficSourceID", "SearchEngineID", "AdvEngineID", "Referer", "URL"]),
    (40, [("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0), ("RefererHash", "=", "@RefererHash"),
          ("TraficSourceID", "in", (-1, 6))] + _JULY, ["URLHash", "EventDate"]),
    (41, [("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0), ("DontCountHits", "=", 0), ("URLHash", "=", "@URLHash")] + _JULY,
     ["WindowClientWidth", "WindowClientHeight"]),
    (42, [("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0), ("DontCountHits", "=", 0),
          ("EventDate", ">=", D(2013, 7, 14)), ("EventDate", "<=", D(2013, 7, 15))], ["EventTime"]),
]
NOTES = {23: "SELECT *: the eight sampled columns stand for the 105", 40: "TraficSourceID IN (-1, 6): evaluated with Arrow on the host "
         "(no InListExpr in LiquidExpr::try_new)"}


def columns_used():
    used = []
    for _q, conj, proj in QUERIES:
        for c in [c for c, _o, _l in conj] + list(proj):
            if c not in used:
                used.append(c)
    return used


def resolve_literals(sample):
    """`@Column` -> a value that occurs in the sample (the most frequent one: a selective but non-empty conjunct)."""
    return {"@" + c: sample.most_frequent(c) for c in ("UserID", "CounterID", "RefererHash", "URLHash")}


def make_expr(column, op, literal, column_type):
    """The PhysicalExpr DataFusion hands to LiquidExpr::try_new for this conjunct (EventDate arrives under its casts:
    `"EventDate"::INT::DATE`, UInt16 -> Int32 -> Date32)."""
    import pyarrow as pa

    from liquid_cache_b200 import BinaryExpr, CastExpr, Column, LikeExpr, Literal

    col = Column(column, 0)
    if op in ("like", "not like"):
        return LikeExpr(op == "not like", False, col, Literal(literal))
    if column == "EventDate":
        col = CastExpr(CastExpr(col, pa.int32()), pa.date32())
    return BinaryExpr(col, op, Literal(literal))


def arrow_mask(arr, op, literal):
    """The Arrow answer for one conjunct on one array (parity check and the host fallback)."""
    import pyarrow as pa
    import pyarrow.compute as pc

    if op == "like":
        return pc.match_like(arr, literal)
    if op == "not like":
        return pc.invert(pc.match_like(arr, literal))
    if op == "in":
        return pc.is_in(arr, value_set=pa.array(list(literal), arr.type))
    if isinstance(literal, dt.date):  # "EventDate"::INT::DATE against a date: compare day numbers
        literal = (literal - dt.date(1970, 1, 1)).days
    fn = {"=": pc.equal, "!=": pc.not_equal, ">=": pc.greater_equal, "<=": pc.less_equal, "<": pc.less, ">": pc.greater}[op]
    return fn(arr, pa.scalar(literal, arr.type))


def run_sweep(cache, rows: int, steps: int, warmup: int, rank: int = 0, world: int = 1, device=None, check_batches: int = 64,
              timer=None, log=None, peak_gbs: float = 0.0):
    """Inserts the shard, runs every query `warmup + steps` times, returns the result dict (rank-local; the caller
    reduces over ranks). `timer()` returns a callable pair (start, stop->ms) — CUDA events in bench.py, perf_counter in tests."""
    import numpy as np
    import pyarrow as pa

    from liquid_cache_b200 import CacheExpression, Column, InListExpr, LiquidExpr, Literal, parquet_array_id
    from liquid_cache_b200 import _native as N
    from synth.hits import HitsSample

    sample = HitsSample()
    lits = resolve_literals(sample)
    cols = columns_used()
    col_id = {c: i for i, c in enumerate(sample.table.column_names)}
    n_entries = max(1, rows // ROWS_PER_ENTRY)
    first = rank * n_entries
    ids = {c: [] for c in cols}
    types = {c: sample.cols[c].type for c in cols}
    def conjunct_literal(lit):
        return lits[lit] if isinstance(lit, str) and lit.startswith("@") else lit

    distinct_conj = {}
    for _q, conj, _proj in QUERIES:
        if conj:
            distinct_conj.setdefault(repr(conj), conj)
    expected = {k: np.zeros(n_entries, dtype=np.int64) for k in distinct_conj}
    t_setup = time.perf_counter()
    insert_s = {"int": 0.0, "str": 0.0}
    group = 512
    for g0 in range(0, n_entries, group):
        nb = min(group, n_entries - g0)
        batches = sample.batches(cols, first + g0, nb)
        for c in cols:
            eids = [parquet_array_id(3, (first + g0 + i) // 32, col_id[c], (first + g0 + i) % 32) for i in range(nb)]
            t0 = time.perf_counter()
            if pa.types.is_string(types[c]):
                # every string column is cached under the SubstringSearch hint; the whole group in one call
                cache.insert_many(eids, batches[c], hint=CacheExpression.SubstringSearch)
                insert_s["str"] += time.perf_counter() - t0
            else:
                cache.insert_many(eids, batches[c])
                insert_s["int"] += time.perf_counter() - t0
            ids[c].extend(int(e) for e in eids)
        # parity data: Arrow's survivor counts per batch for every distinct conjunct list, computed on the very arrays that were
        # inserted, while they are at hand (check_batches >= the shard = every batch of the shard is checked)
        m = min(nb, max(0, check_batches - g0))
        if m:
            for key, conj in distinct_conj.items():
                want = np.ones((m, ROWS_PER_ENTRY), dtype=bool)
                for column, op, lit in conj:
                    mk = arrow_mask(pa.concat_arrays(batches[column][:m]), op, conjunct_literal(lit))
                    want &= np.asarray(mk.fill_null(False).to_numpy(zero_copy_only=False), dtype=bool).reshape(m, ROWS_PER_ENTRY)
                expected[key][g0:g0 + m] = want.sum(axis=1)
    setup_s = time.perf_counter() - t_setup
    handles = {c: cache.handles(ids[c]) for c in cols}
    col_bytes = {c: (sum(int(N.lib().lc_memory_size(cache._ctx, int(h))) for h in handles[c]) if hasattr(cache, "_ctx") else 0) for c in cols}
    rows_local = n_entries * ROWS_PER_ENTRY
    rows_arr = np.full(n_entries, ROWS_PER_ENTRY, dtype=np.uint64)
    scan = cache.scan(rows_arr)
    n_check = min(check_batches, n_entries)

    def host_fallback(column, op, lit):
        """column.rs:143-151: decode the selected rows of every batch, evaluate with Arrow, write the selection back — one
        download of the running selection, one get, one upload (lc_scan_store_selections / lc_scan_load_selections)."""
        if not hasattr(scan, "store_selections"):  # the CPU test double
            counts, _total = scan.counts()
            vals = scan.read(handles[column])
            mask = np.asarray(arrow_mask(vals, op, lit).fill_null(False).to_numpy(zero_copy_only=False), dtype=bool)
            pos = 0
            for b in range(n_entries):
                k = int(counts[b])
                sel = np.asarray(scan.selection(b).to_numpy(zero_copy_only=False), dtype=bool)
                new = np.zeros(ROWS_PER_ENTRY, dtype=bool)
                new[np.flatnonzero(sel)] = mask[pos:pos + k]
                pos += k
                scan.set_selection(b, new)
            return
        words = np.array(scan.store_selections(), dtype=np.uint32)  # a private copy: the surviving words are edited below
        nz = np.flatnonzero(words)
        if len(nz) == 0:
            return  # nothing selected any more: nothing to decode or evaluate (liquid_cache_reader.rs:308-311)
        vals = scan.read(handles[column])  # rows in batch order, then row order: the order of the set bits below
        mask = np.asarray(arrow_mask(vals, op, lit).fill_null(False).to_numpy(zero_copy_only=False), dtype=bool)
        # only the words that still have a bit set are unpacked (a selection behind earlier conjuncts is mostly zero words;
        # unpacking all 16.8 M bits cost 30 ms per call)
        bits = np.unpackbits(words[nz].view(np.uint8).reshape(len(nz), 4), axis=1, bitorder="little").reshape(-1)
        set_pos = np.flatnonzero(bits)
        assert len(set_pos) == len(mask)
        bits[set_pos[~mask]] = 0
        words[nz] = np.packbits(bits.reshape(len(nz), 32), axis=1, bitorder="little").view(np.uint32).reshape(-1)
        scan.load_selections(words)

    # q40's IN conjunct is also run as a device filter (LC_OP_IN) when the scan evaluates InListExpr: the native scan does
    # (`filter_native` is the sign of it); the comparison / LIKE-only CPU test double does not
    device_in = hasattr(scan, "filter_native")
    trace_q = os.environ.get("LC_SWEEP_TRACE")  # diagnosis: wall clock per conjunct of one query (synchronises after each)

    def run_query(conj, proj, to_host, want_counts=False, q=None, in_on_device=False):
        scan.reset()
        for column, op, lit in conj:
            lit = conjunct_literal(lit)
            t_c = time.perf_counter()
            if op == "in" and in_on_device:
                # the same conjunct as a device InListExpr (LC_OP_IN): the reference's LiquidExpr would refuse it
                expr = LiquidExpr.new_unchecked(InListExpr(Column(column, 0), tuple(Literal(v) for v in lit)))
                scan.filter(handles[column], expr, types[column])
            elif op == "in":
                host_fallback(column, op, lit)
            else:
                expr = LiquidExpr.try_new(make_expr(column, op, lit, types[column]), types[column], CacheExpression.SubstringSearch)
                scan.filter(handles[column], expr, types[column])
            if trace_q is not None and q is not None and str(q) == trace_q:
                cache.synchronize()
                print(f"[sweep trace] q{q} {column} {op}: {1e3 * (time.perf_counter() - t_c):.3f} ms, {scan.counts()[1]} rows left", file=sys.stderr)
        out = []
        counts, total = None, None
        if want_counts or not proj or not conj:
            counts, total = scan.counts()  # COUNT(*)-shaped queries need the survivor count itself; so does the parity check
        if not conj or total is None or total:
            for c in proj:
                if to_host:
                    out.append(scan.read(handles[c]))  # after a filter: planned on the device, one synchronisation
                else:
                    r = scan.read_torch_borrowed(handles[c], device) if conj else None  # no filter: a plain full-column decode
                    out.append(r if r is not None else scan.read_torch(handles[c], device))
        if total is None:
            first_out = out[0]
            total = len(first_out) if (to_host or not isinstance(first_out, tuple)) else int(first_out[2] if len(first_out) == 3 else first_out[3])
        return counts, total, out

    def safe(fn):
        """A get whose decoded bytes pass 2 GiB (int32 offsets of Utf8) is refused by the library: note it, keep sweeping."""
        try:
            return fn(), None
        except N.NativeError as e:
            return None, str(e)

    results = []
    for q, conj, proj in QUERIES:
        if not conj and not proj:
            results.append({"q": q, "ms": 0.0, "e2e_ms": 0.0, "rows_out": rows_local, "note": "no column touched"})
            continue
        first, err = safe(lambda: run_query(conj, proj, False, want_counts=True, q=q))
        if err:
            results.append({"q": q, "ms": 0.0, "e2e_ms": 0.0, "rows_out": 0, "note": "not run: " + err})
            continue
        for _ in range(max(0, warmup - 1)):
            run_query(conj, proj, False)
        counts, total, _ = first
        # parity on the first batches: survivor counts against Arrow on the very arrays that were inserted
        ok = True
        if conj:
            ok = bool(np.array_equal(np.asarray(counts[:n_check], dtype=np.int64), expected[repr(conj)][:n_check]))
        ms = []
        for _ in range(steps):
            start, stop = timer()
            start()
            run_query(conj, proj, False)
            ms.append(stop())
        e2e = []
        for _ in range(max(1, steps // 2)):
            t0 = time.perf_counter()
            run_query(conj, proj, True)
            e2e.append((time.perf_counter() - t0) * 1e3)
        pred_cols = []
        for column, _o, _l in conj:
            if column not in pred_cols:
                pred_cols.append(column)
        pred_bytes = sum(col_bytes[c] for c in pred_cols)
        # projected columns are read only where rows survive: batches without survivors are never touched
        hit_frac = float(np.count_nonzero(np.asarray(counts)) / n_entries) if conj else 1.0
        proj_bytes = int(sum(col_bytes[c] for c in proj) * hit_frac) if (total or not conj) else 0
        sel_bytes = (rows_local // 8) * max(0, 2 * len(conj) - 1)  # running selection: written by the first conjunct, read + written after
        med_ms = float(np.median(ms))
        touched = pred_bytes + proj_bytes + sel_bytes
        r = {"q": q, "ms": med_ms, "e2e_ms": float(np.median(e2e)), "rows_out": int(total), "selectivity": int(total) / rows_local,
             "conjuncts": len(conj), "projected": len(proj), "counts_match_arrow": ok, "batches_checked": n_check,
             "predicate_column_bytes": pred_bytes, "projected_column_bytes_read": proj_bytes,
             "roofline": {"bound": "hbm", "algorithmic_bytes": touched, "achieved": touched / (med_ms / 1e3) / 1e9 if med_ms else 0.0,
                          "unit": "GB/s", "peak": peak_gbs, "frac": (touched / (med_ms / 1e3) / 1e9 / peak_gbs) if (med_ms and peak_gbs) else None,
                          "note": "liquid bytes of the predicate columns + of the projected columns in batches with survivors + the "
                                  "running selection, over the query's device time (all launches, host gaps included)"}}
        if q in NOTES:
            r["note"] = NOTES[q]
        if device_in and any(op == "in" for _c, op, _l in conj):
            # the IN conjunct on the device as well (the host path above stays, so the sweep totals compare with earlier runs)
            d_counts, d_total, _ = run_query(conj, proj, False, want_counts=True, in_on_device=True)
            d_ok = bool(np.array_equal(np.asarray(d_counts[:n_check], dtype=np.int64), expected[repr(conj)][:n_check]))
            d_ms = []
            for _ in range(steps):
                start, stop = timer()
                start()
                run_query(conj, proj, False, in_on_device=True)
                d_ms.append(stop())
            d_e2e = []
            for _ in range(max(1, steps // 2)):
                t0 = time.perf_counter()
                run_query(conj, proj, True, in_on_device=True)
                d_e2e.append((time.perf_counter() - t0) * 1e3)
            r["device_in_list"] = {"ms": float(np.median(d_ms)), "e2e_ms": float(np.median(d_e2e)), "rows_out": int(d_total),
                                   "counts_match_arrow": d_ok}
        results.append(r)
        if log:
            log(f"q{q}: {r['ms']:.3f} ms device, {r['e2e_ms']:.3f} ms e2e, {total} rows, parity {ok}")
    scan.close()
    total_ms = sum(r["ms"] for r in results)
    total_e2e = sum(r["e2e_ms"] for r in results)
    # the same totals with the device IN-list variant in place of the host path
    total_ms_dev = sum(r["device_in_list"]["ms"] if "device_in_list" in r else r["ms"] for r in results)
    total_e2e_dev = sum(r["device_in_list"]["e2e_ms"] if "device_in_list" in r else r["e2e_ms"] for r in results)
    touched = [r for r in results if r.get("conjuncts", 0) + r.get("projected", 0) > 0]
    return {"rows_local": rows_local, "n_entries": n_entries, "setup_seconds": setup_s, "insert_seconds": insert_s, "queries": results,
            "sweep_ms": total_ms, "sweep_e2e_ms": total_e2e, "sweep_ms_device_in_list": total_ms_dev,
            "sweep_e2e_ms_device_in_list": total_e2e_dev, "queries_touching_columns": len(touched),
            "all_counts_match_arrow": all(r.get("counts_match_arrow", True) and r.get("device_in_list", {}).get("counts_match_arrow", True)
                                          for r in results),
            "literals_from_sample": {k: int(v) for k, v in lits.items()}}


def main(args, rank, world, local_rank):
    """Entry point used by bench.py: one JSON line; metric = rows scanned by the sweep per second (every query that touches a
    column scans the whole shard once), device-resident and end to end."""
    import numpy as np
    import torch
    import torch.distributed as dist

    import bench
    from liquid_cache_b200 import LiquidCacheBuilder

    torch.cuda.set_device(local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    cache = LiquidCacheBuilder.new().with_device(local_rank).build()
    stream = torch.cuda.Stream(device=local_rank)
    torch.cuda.set_stream(stream)
    cache.set_stream(stream.cuda_stream)

    def timer():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def stop():
            e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1)

        return (lambda: e0.record(stream)), stop

    rows = args.rows if args.rows != 100_000_000 else 16_777_216  # 2048 entries per column; a full URL get stays under 2 GiB
    clocks = bench.ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    peak0, _src0 = bench.measured_peak_gbs()
    check = 1 << 30 if os.environ.get("LC_SWEEP_CHECK_ALL") == "1" else 64  # every batch of the shard, or the first 64
    res = run_sweep(cache, rows, max(3, args.steps // 4), max(3, args.warmup), rank, world, torch.device("cuda", local_rank), timer=timer,
                    check_batches=check, peak_gbs=peak0,
                    log=(lambda s: print(s, file=sys.stderr)) if rank == 0 and os.environ.get("LC_BENCH_TRACE") == "1" else None)
    t = torch.tensor([res["sweep_ms"], res["sweep_e2e_ms"]], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    sweep_ms, sweep_e2e = [float(x) for x in t.tolist()]
    clk = clocks.stop() if rank == 0 else None
    if rank == 0:
        scanned = res["rows_local"] * world * res["queries_touching_columns"]
        peak, peak_src = bench.measured_peak_gbs()
        slow = sorted(res["queries"], key=lambda r: -r["ms"])[:5]
        line = {
            "metric": "filtered-scan Mrows/s (ClickBench 43-query scan sweep, hot cache)", "value": scanned / (sweep_ms / 1e3) / 1e6,
            "unit": "Mrows/s", "n_gpus": world, "steps": max(3, args.steps // 4), "warmup": max(3, args.warmup), "ms_per_step": sweep_ms,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            "config": {"workload": "scan stage of ClickBench q0-q42 (conjuncts refine the selection on the device, projected columns read "
                                   "with the final selection) over a hits-shaped shard resampled from the 24 586-row ClickBench sample "
                                   "(BASELINE configs[4])",
                       "rows_per_gpu": res["rows_local"], "entries_per_gpu_per_column": res["n_entries"], "columns": len(columns_used()),
                       "liquid_bytes_per_gpu": int(cache.stats().hbm_bytes_used), "setup_seconds": res["setup_seconds"],
                       "insert_seconds": res["insert_seconds"], "all_counts_match_arrow": res["all_counts_match_arrow"],
                       "batches_checked_against_arrow": min(check, res["n_entries"]),
                       "literals_from_sample": res["literals_from_sample"], "slowest_queries": [{"q": r["q"], "ms": r["ms"]} for r in slow],
                       "parallelism": f"entries sharded by EntryID over {world} GPU(s), no data-path collective"},
            "e2e": {"value": scanned / (sweep_e2e / 1e3) / 1e6, "unit": "Mrows/s", "ms_per_step": sweep_e2e},
            # rank 0's totals with q40's IN conjunct evaluated on the device instead of by the host path
            "device_in_list": {"ms_per_step": res["sweep_ms_device_in_list"], "e2e_ms_per_step": res["sweep_e2e_ms_device_in_list"]},
            "queries": res["queries"], "peak_source": peak_src, "hbm_peak_gbs": peak, "clocks": clk,
        }
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    cache.close()
