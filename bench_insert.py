"""`bench.py --workload insert`: the FIRST half of the path — transcoding Arrow batches into liquid columns on insert()
(cache/transcode.rs:46-290; byte views conversions.rs:260-373, integers primitive_array.rs:159-206) — timed by itself.

Input: Arrow batches whose buffers are PAGE-LOCKED host memory (what a reader that means to feed a GPU cache would decode
into), so the library uploads straight from them. One step = `lc_cache_insert_many` over a group of batches; the timed
region holds the H2D copies, the encode kernels and the blob layout. Reported per column:
  Mrows/s, Arrow GB/s in, liquid GB/s out, and the two rooflines the step can hit — PCIe (Arrow bytes in / measured
  pinned H2D bandwidth) and HBM ((Arrow in + liquid out) / measured copy peak) — plus the CPU arm: the C port of the
  reference's transcode (oracle/c: dictionary + FSST + prefix keys + fingerprints, FoR + FastLanes pack) on the host
  threads the container may use.
"""
from __future__ import annotations

import concurrent.futures as cf
import json
import os
import time

ROWS_PER_ENTRY = 8192


def _pinned_copy(arr, torch, keep):
    """The same Arrow array with every buffer in page-locked memory."""
    import pyarrow as pa

    bufs = []
    for b in arr.buffers():
        if b is None:
            bufs.append(None)
            continue
        t = torch.empty(max(b.size, 1), dtype=torch.uint8, pin_memory=True)
        t[: b.size] = torch.frombuffer(b, dtype=torch.uint8)
        keep.append(t)
        bufs.append(pa.foreign_buffer(t.data_ptr(), b.size, base=t))
    return pa.Array.from_buffers(arr.type, len(arr), bufs, null_count=arr.null_count, offset=arr.offset)


def h2d_peak_gbs(torch, device, nbytes=256 << 20):
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device=device)
    best = 0.0
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        best = max(best, nbytes / (e0.elapsed_time(e1) / 1e3) / 1e9)
    return best


def cpu_transcode(column: str, arrays, threads: int, target_s: float = 4.0):
    """The reference's transcode on the CPU (C port), batches spread over `threads` workers; strings train one FSST table
    per 32 batches (a row group's column chunk, transcode.rs:16-33)."""
    from oracle import c_oracle as CO

    CO.lib()
    is_str = column == "URL"

    def run_group(g):
        if is_str:
            fsst = CO.CFsst(g[0])
            return [CO.CStrArray(a, fsst, build_fingerprints=True) for a in g]
        return [CO.CIntArray(a) for a in g]

    groups = [arrays[i:i + 32] for i in range(0, len(arrays), 32)]
    rows = sum(len(a) for a in arrays)
    with cf.ThreadPoolExecutor(threads) as ex:
        list(ex.map(run_group, groups[: max(1, threads)]))  # warm-up
        reps, t0 = 0, time.perf_counter()
        while True:
            list(ex.map(run_group, groups))
            reps += 1
            dt = time.perf_counter() - t0
            if dt >= target_s:
                break
    return {"value": rows * reps / dt / 1e6, "unit": "Mrows/s", "cores": threads, "kind": "port",
            "sample": f"{len(arrays)} batches x {ROWS_PER_ENTRY} rows of {column}, {reps} passes in {dt:.1f} s; oracle/c encode "
                      f"(dictionary + FSST + prefix keys + fingerprints / FoR + FastLanes pack), {threads} threads over row groups"}


def main(args, rank, world, local_rank):
    import numpy as np
    import pyarrow as pa
    import torch

    import bench_cpu
    import synth
    from liquid_cache_b200 import CacheExpression, EntryID, LiquidCacheBuilder, parquet_array_id

    from bench import measured_peak_gbs

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    cache = LiquidCacheBuilder.new().with_device(local_rank).build()
    stream = torch.cuda.Stream(device=local_rank)
    torch.cuda.set_stream(stream)
    cache.set_stream(stream.cuda_stream)
    pcie = h2d_peak_gbs(torch, dev)
    hbm, hbm_src = measured_peak_gbs()
    threads, host = bench_cpu.usable_cpus()
    n_batches = max(64, min(args.rows, 16_777_216) // ROWS_PER_ENTRY)  # per column; 2048 batches = 16.8 M rows by default
    synth.lib().lcs_init(synth.URL_POOL)
    columns = [("URL", 13, 256, CacheExpression.SubstringSearch), ("EventTime", 4, 1024, None), ("UserID", 9, 1024, None),
               ("l_shipdate", 10, 1024, None)]
    out = []
    for name, col_id, group, hint in columns:
        keep = []
        with cf.ThreadPoolExecutor(min(32, threads * 2)) as ex:
            if name == "URL":
                raw = list(ex.map(synth.url_entry, range(n_batches)))
            elif name == "l_shipdate":
                raw = list(ex.map(lambda i: synth.int_entry("l_shipdate", i, seed=synth.SEED_TPCH), range(n_batches)))
            else:
                raw = list(ex.map(lambda i: synth.int_entry(name, i), range(n_batches)))
        arrays = [_pinned_copy(a, torch, keep) for a in raw]
        arrow_bytes = sum(a.nbytes for a in arrays)
        ids = [parquet_array_id(1, i // 32, col_id, i % 32) for i in range(n_batches)]

        def one_pass():
            for g0 in range(0, n_batches, group):
                cache.insert_many([EntryID(int(x)) for x in ids[g0:g0 + group]], arrays[g0:g0 + group], hint=hint)

        steps = max(2, min(args.steps, 5))
        for _ in range(2):  # warm-up: scratch grows to its size, symbol tables of every row group are trained ONCE here ...
            one_pass()
        cache.synchronize()
        st0 = cache.stats()
        t0 = time.perf_counter()
        for _ in range(steps):  # ... so the timed passes re-insert (replace) every batch with the tables in place
            one_pass()
        cache.synchronize()
        dt = (time.perf_counter() - t0) / steps
        st1 = cache.stats()
        liquid_bytes = int(st1.hbm_bytes_used)  # this column's entries (the previous column was reset)
        rows = n_batches * ROWS_PER_ENTRY
        line = {"column": name, "Mrows_per_s": rows / dt / 1e6, "ms_per_pass": dt * 1e3, "batches": n_batches, "batches_per_call": group,
                "arrow_bytes_in": arrow_bytes, "liquid_bytes_out": liquid_bytes, "arrow_GB_per_s": arrow_bytes / dt / 1e9,
                "h2d_bytes_per_pass": int((st1.h2d_bytes - st0.h2d_bytes) / steps),
                "gpu_launches_per_pass": int((st1.kernel_launches - st0.kernel_launches) / steps),
                "roofline": {"pcie": {"achieved": arrow_bytes / dt / 1e9, "peak": pcie, "unit": "GB/s", "frac": arrow_bytes / dt / 1e9 / pcie,
                                      "peak_source": "pinned host -> device copy of 256 MB measured in this run"},
                             "hbm": {"achieved": (arrow_bytes + liquid_bytes) / dt / 1e9, "peak": hbm, "unit": "GB/s",
                                     "frac": (arrow_bytes + liquid_bytes) / dt / 1e9 / hbm, "peak_source": hbm_src}}}
        if not args.no_cpu_baseline and rank == 0:
            sample = raw[: min(len(raw), 32 * max(8, threads))]
            line["cpu_baseline"] = cpu_transcode(name, sample, threads)
            line["cpu_baseline"]["host"] = host
        out.append(line)
        cache.reset()
        del arrays, keep, raw
    print(json.dumps({
        "metric": "insert() transcode Mrows/s (Arrow batches in page-locked host memory -> liquid columns in HBM)", "unit": "Mrows/s",
        "value": float(np.mean([c["Mrows_per_s"] for c in out])), "n_gpus": 1, "steps": args.steps, "warmup": 2, "higher_is_better": True,
        "data": "synthetic", "dtype": "u8/int64", "config": {"workload": "insert / transcode of the bench columns", "rows_per_column": n_batches * ROWS_PER_ENTRY},
        "columns": out}))
    cache.close()
