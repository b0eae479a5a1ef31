"""Disjunctions over columns in the device scan (lc_scan_filter_or) against the reference-shaped host path, on the same
16.8 M-row hits shard as bench_sweep.py (2048 batches of 8192 rows per column). Prints one JSON line.

Per query, two paths, each checked against Arrow's survivor count on EVERY batch:
  device  ordinary conjuncts with lc_scan_filter, the OR with ONE lc_scan_filter_or; the selection never leaves HBM
  host    CachedRowGroup::evaluate_selection_with_predicate (src/datafusion/src/cache/mod.rs:111-150): the running selection
          is downloaded, every leaf is evaluated on the encoded data under it (lc_eval_predicate_many), the masks are joined
          with or_kleene on the host and the selection is uploaded again. An OR of AND groups has no such path in the
          reference: its involved columns are decoded under the selection, pyarrow evaluates the tree, the result is loaded back.
Times are CUDA events on the scan's stream around the whole query (host work of the host path included), median of --steps.

    python bench_or.py [--steps 5] [--warmup 2] [--rows 16777216]
"""
from __future__ import annotations

import argparse
import datetime as dt
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_sweep import ROWS_PER_ENTRY, arrow_mask, make_expr, resolve_literals  # noqa: E402

D = dt.date
_JULY = [("EventDate", ">=", D(2013, 7, 1)), ("EventDate", "<=", D(2013, 7, 31))]
# (name, ordinary conjuncts, OR of AND groups, projected columns)
QUERIES = [
    ("a", [], [[("URL", "like", "%google%")], [("Referer", "like", "%google%")]], []),
    ("b", [], [[("SearchPhrase", "!=", "")], [("MobilePhoneModel", "!=", "")]], []),
    ("c", [], [[("AdvEngineID", "!=", 0)], [("TraficSourceID", "in", (-1, 6))]], []),
    ("d", [], [[("CounterID", "=", "@CounterID"), ("IsRefresh", "=", 0)], [("URLHash", "=", "@URLHash")]], []),
    ("e", _JULY, [[("IsLink", "!=", 0)], [("IsDownload", "!=", 0)]], ["URL"]),
]


def columns_used():
    used = []
    for _n, conj, dnf, proj in QUERIES:
        for c in [c for c, _o, _l in conj] + [c for d in dnf for c, _o, _l in d] + list(proj):
            if c not in used:
                used.append(c)
    return used


def card():
    """(name, power limit in W) of the GPU the benchmark runs on, read in the same run."""
    import torch

    name, limit = torch.cuda.get_device_name(0), None
    try:
        idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rows", type=int, default=16_777_216)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc
    import torch

    from liquid_cache_b200 import (CacheExpression, Column, InListExpr, LiquidCacheBuilder, LiquidExpr, Literal,
                                   parquet_array_id)
    from synth.hits import HitsSample

    torch.cuda.set_device(0)
    cache = LiquidCacheBuilder.new().with_device(0).build()
    stream = torch.cuda.Stream(device=0)
    torch.cuda.set_stream(stream)
    cache.set_stream(stream.cuda_stream)
    device = torch.device("cuda", 0)

    sample = HitsSample()
    lits = resolve_literals(sample)
    lit_of = lambda v: lits[v] if isinstance(v, str) and v.startswith("@") else v  # noqa: E731
    cols = columns_used()
    col_id = {c: i for i, c in enumerate(sample.table.column_names)}
    types = {c: sample.cols[c].type for c in cols}
    n_entries = max(1, args.rows // ROWS_PER_ENTRY)
    ids = {c: [] for c in cols}
    expected = {name: np.zeros(n_entries, dtype=np.int64) for name, *_ in QUERIES}

    def fill(m):
        return np.asarray(m.fill_null(False).to_numpy(zero_copy_only=False), dtype=bool)

    t_setup = time.perf_counter()
    for g0 in range(0, n_entries, 512):
        nb = min(512, n_entries - g0)
        batches = sample.batches(cols, g0, nb)
        for c in cols:
            eids = [parquet_array_id(5, (g0 + i) // 32, col_id[c], (g0 + i) % 32) for i in range(nb)]
            if pa.types.is_string(types[c]):
                cache.insert_many(eids, batches[c], hint=CacheExpression.SubstringSearch)
            else:
                cache.insert_many(eids, batches[c])
            ids[c].extend(int(e) for e in eids)
        whole = {c: pa.concat_arrays(batches[c]) for c in cols}
        for name, conj, dnf, _proj in QUERIES:  # Arrow's survivor count of every batch
            want = np.ones(nb * ROWS_PER_ENTRY, dtype=bool)
            for c, op, lit in conj:
                want &= fill(arrow_mask(whole[c], op, lit_of(lit)))
            acc = np.zeros_like(want)
            for d in dnf:
                m = np.ones_like(want)
                for c, op, lit in d:
                    m &= fill(arrow_mask(whole[c], op, lit_of(lit)))
                acc |= m
            expected[name][g0:g0 + nb] = (want & acc).reshape(nb, ROWS_PER_ENTRY).sum(axis=1)
    setup_s = time.perf_counter() - t_setup
    handles = {c: cache.handles(ids[c]) for c in cols}
    rows_arr = np.full(n_entries, ROWS_PER_ENTRY, dtype=np.uint64)
    scan = cache.scan(rows_arr)
    word_off, _total = scan.selection_layout()
    n_words = (ROWS_PER_ENTRY + 31) // 32

    def leaf(c, op, lit):
        lit = lit_of(lit)
        if op == "in":
            return LiquidExpr.new_unchecked(InListExpr(Column(c, 0), tuple(Literal(v) for v in lit)))
        return LiquidExpr.try_new(make_expr(c, op, lit, types[c]), types[c], CacheExpression.SubstringSearch)

    def host_or(dnf):
        """The reference-shaped path for the OR conjunct (see the module docstring)."""
        words = np.array(scan.store_selections(), dtype=np.uint32)
        nz = np.flatnonzero(words)
        if len(nz) == 0:
            return
        bits = np.unpackbits(words[nz].view(np.uint8).reshape(len(nz), 4), axis=1, bitorder="little").reshape(-1)
        set_pos = np.flatnonzero(bits)
        if all(len(d) == 1 for d in dnf):
            # every leaf on the encoded data under the same selection, or_kleene of the masks
            sels = [words[int(o):int(o) + n_words].view(np.uint8) for o in word_off]
            combined = None
            for (c, op, lit), in dnf:
                vals, valid, offs, out_len, _nulls, _t = cache.eval_predicate_many(handles[c], rows_arr, leaf(c, op, lit), types[c], sels)
                # batch i's mask is out_len[i] bits from byte offs[i]: one gather over the unpacked buffers
                lens = out_len.astype(np.int64)
                idx = np.repeat(offs.astype(np.int64) * 8 - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
                v_bits = np.unpackbits(vals, bitorder="little")[idx].astype(bool)
                ok = np.unpackbits(valid, bitorder="little")[idx].astype(bool)  # written for every batch, all ones without nulls
                mask = pa.array(v_bits, mask=~ok)
                combined = mask if combined is None else pc.or_kleene(combined, mask)
            keep = fill(combined)
        else:
            # no encoded-data path for an OR of AND groups: decode the involved columns under the selection, let Arrow decide
            decoded = {}
            for d in dnf:
                for c, _op, _lit in d:
                    if c not in decoded:
                        decoded[c] = scan.read(handles[c])
            keep = np.zeros(len(set_pos), dtype=bool)
            for d in dnf:
                m = np.ones(len(set_pos), dtype=bool)
                for c, op, lit in d:
                    m &= fill(arrow_mask(decoded[c], op, lit_of(lit)))
                keep |= m
        assert len(keep) == len(set_pos)
        bits[set_pos[~keep]] = 0
        words[nz] = np.packbits(bits.reshape(len(nz), 32), axis=1, bitorder="little").view(np.uint32).reshape(-1)
        scan.load_selections(words)

    def run(conj, dnf, proj, path):
        scan.reset()
        for c, op, lit in conj:
            scan.filter(handles[c], leaf(c, op, lit), types[c])
        if path == "device":
            scan.filter_or([[(handles[c], leaf(c, op, lit), types[c]) for c, op, lit in d] for d in dnf])
        else:
            host_or(dnf)
        counts, total = scan.counts()
        if total:
            for c in proj:
                r = scan.read_torch_borrowed(handles[c], device)
                if r is None:
                    scan.read_torch(handles[c], device)
        return counts, total

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    results = []
    for name, conj, dnf, proj in QUERIES:
        r = {"q": name, "or": " OR ".join("(" + " AND ".join(f"{c} {op} {lit_of(lit)!r}" for c, op, lit in d) + ")" for d in dnf),
             "conjuncts_before": len(conj), "projected": proj}
        for path in ("device", "host"):
            counts, total = run(conj, dnf, proj, path)
            ok = bool(np.array_equal(np.asarray(counts, dtype=np.int64), expected[name]))
            for _ in range(max(0, args.warmup - 1)):
                run(conj, dnf, proj, path)
            ms = [timed(lambda: run(conj, dnf, proj, path)) for _ in range(args.steps)]
            r[path] = {"ms": float(np.median(ms)), "rows_out": int(total), "counts_match_arrow": ok, "batches_checked": n_entries}
        r["host_over_device"] = r["host"]["ms"] / r["device"]["ms"] if r["device"]["ms"] else None
        results.append(r)
    scan.close()
    gpu, limit = card()
    print(json.dumps({
        "metric": "OR conjunct over columns: device (lc_scan_filter_or) vs host round trip, ms per query (median)",
        "gpu": gpu, "power_limit_w": limit, "rows": n_entries * ROWS_PER_ENTRY, "batches": n_entries, "steps": args.steps,
        "warmup": args.warmup, "setup_seconds": setup_s, "literals_from_sample": {k: int(v) for k, v in lits.items()},
        "all_counts_match_arrow": all(r[p]["counts_match_arrow"] for r in results for p in ("device", "host")),
        "queries": results,
    }))
    cache.close()


if __name__ == "__main__":
    main()
