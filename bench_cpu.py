"""The timed CPU arm of bench.py (`cpu_baseline` and `--impl reference`): the C port of the reference's CPU path
(oracle/c/lc_oracle.c) driven the way the reference is driven — a fixed set of worker threads created once (tokio's
runtime; DataFusion partition tasks over `LiquidCacheReader`, src/datafusion/src/reader/runtime/liquid_cache_reader.rs:297-391)
that take batches of the scan. Nothing is created, joined or allocated per pass inside the clock, a pass covers at least
64 entries per thread, and the single-thread rate is reported beside the pooled one so the scaling can be checked
(`threads x single` is the ceiling; hyper-threads do not double it).

This is bench infrastructure: it is the only module besides tests/ and __graft_entry__.smoke() that touches oracle/.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import time

ROWS_PER_ENTRY = 8192


def physical_cores() -> int:
    try:
        import psutil

        return int(psutil.cpu_count(logical=False) or os.cpu_count() or 1)
    except Exception:
        return os.cpu_count() or 1


def usable_cpus() -> tuple[int, dict]:
    """Threads the CPU arm should run: the logical CPUs this process may use, capped by the container's CPU quota
    (cgroup v2 cpu.max / v1 cfs quota). A container may see far more logical CPUs than its quota grants; threads beyond
    the quota are throttled, so asking for more of them makes the baseline slower, not faster."""
    logical = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    quota = None
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            quota = float(q) / float(per)
    except (OSError, ValueError):
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except (OSError, ValueError):
            pass
    threads = logical if quota is None else max(1, min(logical, int(quota + 0.5)))
    return threads, {"logical_cpus": logical, "cgroup_cpu_quota": quota, "threads_used": threads}


def default_sample_entries(threads: int, cap: int) -> int:
    """>= 64 entries per thread per pass (VERDICT r1 item 1), bounded by the workload's own size."""
    return max(64, min(cap, max(8192, 64 * threads)))


class CpuArm:
    """One workload on the CPU port: entries built in parallel (untimed), a persistent pool, timed passes."""

    def __init__(self, workload: str, sample_entries: int, threads: int, first_entry: int = 0, params: dict | None = None):
        import synth
        from oracle import c_oracle as CO

        CO.lib()  # -march=native: build() runs on the machine that is timed
        self.CO = CO
        self.workload = workload
        self.threads = threads
        self.n = sample_entries
        self.params = dict(params or {})
        build_threads = min(64, max(1, threads))
        t0 = time.perf_counter()
        if workload == "url_like":
            synth.lib().lcs_init(synth.URL_POOL)
            first = synth.url_entry(first_entry)
            fsst = CO.CFsst(first)  # one symbol table per column chunk, trained on the first batch

            def mk(i):
                return CO.CStrArray(synth.url_entry(i), fsst, build_fingerprints=True)

            with cf.ThreadPoolExecutor(build_threads) as ex:
                self.entries = list(ex.map(mk, range(first_entry, first_entry + sample_entries)))
            self._fsst = fsst
            self.needle = self.params.get("needle", b"google")
            self.kind, self.args = 3, (self.needle, 0, 0, 0, 0)
            self.entries2 = None
        elif workload == "shipdate":
            with cf.ThreadPoolExecutor(build_threads) as ex:
                self.entries = list(ex.map(
                    lambda i: CO.CIntArray(synth.int_entry("l_shipdate", i, seed=synth.SEED_TPCH)),
                    range(first_entry, first_entry + sample_entries)))
            self.kind, self.args = 5, (b"", 5, int(self.params["lo_days"]), 2, int(self.params["hi_days"]))  # 5 = GE, 2 = LT
            self.entries2 = None
        elif workload == "int_filter":
            with cf.ThreadPoolExecutor(build_threads) as ex:
                self.entries = list(ex.map(lambda i: CO.CIntArray(synth.int_entry("EventTime", i)),
                                           range(first_entry, first_entry + sample_entries)))
                self.entries2 = list(ex.map(lambda i: CO.CIntArray(synth.int_entry("UserID", i)),
                                            range(first_entry, first_entry + sample_entries)))
            self.kind, self.args = 4, (b"", 5, int(self.params["lo"]), 2, int(self.params["hi"]))
        else:
            raise ValueError(workload)
        self.build_s = time.perf_counter() - t0
        self.pool = CO.ScanPool(threads).bind(self.entries)
        self.pool1 = None
        if self.entries2 is not None:
            self.pool.bind_second(self.entries2, 0, int(self.params["uid"]))  # 0 = EQ
        self.rows_per_pass = sample_entries * ROWS_PER_ENTRY

    def one_pass(self):
        needle, op1, l1, op2, l2 = self.args
        return self.pool.scan(self.kind, needle, op1, l1, op2, l2, grain=4)

    def single_thread_mrows(self, target_s: float = 1.5, entries: int = 256):
        """The same per-entry work on ONE thread over the first `entries` entries (a one-thread pool, same code path)."""
        CO = self.CO
        m = min(entries, self.n)
        if self.pool1 is None:
            self.pool1 = CO.ScanPool(1).bind(self.entries[:m])
            if self.entries2 is not None:
                self.pool1.bind_second(self.entries2[:m], 0, int(self.params["uid"]))
        needle, op1, l1, op2, l2 = self.args
        self.pool1.scan(self.kind, needle, op1, l1, op2, l2, grain=4)
        reps, t0 = 0, time.perf_counter()
        while True:
            _m, rows = self.pool1.scan(self.kind, needle, op1, l1, op2, l2, grain=4)
            reps += 1
            dt = time.perf_counter() - t0
            if dt >= target_s:
                break
        return rows * reps / dt / 1e6

    def timed(self, target_s: float = 8.0, warmup: int = 2, max_reps: int = 100000):
        for _ in range(warmup):
            self.one_pass()
        reps, t0 = 0, time.perf_counter()
        matched = rows = 0
        while True:
            matched, rows = self.one_pass()
            reps += 1
            dt = time.perf_counter() - t0
            if dt >= target_s or reps >= max_reps:
                break
        return {"mrows": rows * reps / dt / 1e6, "reps": reps, "seconds": dt, "matched": matched, "rows": rows,
                "ms_per_pass": dt / reps * 1e3}

    def describe(self, single: float, pooled: float) -> dict:
        phys = physical_cores()
        _t, host = usable_cpus()
        # the ceiling the pooled figure is checked against: what the process can actually get (quota), not what it can see
        ceil_cores = min(self.threads, phys) if host["cgroup_cpu_quota"] is None else min(self.threads, host["cgroup_cpu_quota"])
        return {"threads": self.threads, "threads_physical": phys, "host": host, "single_thread_Mrows_per_s": single,
                "threads_x_single": single * self.threads, "usable_cores_x_single": single * ceil_cores,
                "pooled_over_usable_cores_x_single": pooled / (single * ceil_cores) if single else None,
                "entries_per_thread_per_pass": self.n / self.threads, "entries_per_pass": self.n,
                "pool": "persistent pthreads created once outside the clock, entries handed out 4 at a time "
                        "(oracle/c/lc_oracle.c lco_pool_*)"}

    def close(self):
        self.pool.close()
        if self.pool1 is not None:
            self.pool1.close()


def cpu_baseline_line(workload: str, sample_entries: int, threads: int, params: dict | None = None, target_s: float = 8.0):
    """The `cpu_baseline` object of a bench line."""
    arm = CpuArm(workload, sample_entries, threads, params=params)
    try:
        single = arm.single_thread_mrows()
        t = arm.timed(target_s)
    finally:
        arm.close()
    what = {"url_like": "the same synthetic URL column: LIKE '%google%' + get of the hits",
            "shipdate": "the same l_shipdate column: two range conjuncts + and_then + get of the survivors",
            "int_filter": "the same EventTime / UserID columns: three conjuncts + and_then + get of both columns"}[workload]
    out = {"value": t["mrows"], "unit": "Mrows/s", "cores": threads, "kind": "port",
           "sample": f"{sample_entries} entries x {ROWS_PER_ENTRY} rows of {what}; {t['reps']} passes in {t['seconds']:.1f} s, "
                     f"{t['matched']} rows matched per pass; C restatement of the reference path (oracle/c/lc_oracle.c)",
           "ms_per_pass": t["ms_per_pass"], "rows_per_pass": t["rows"], "setup_seconds": arm.build_s}
    out.update(arm.describe(single, t["mrows"]))
    return out
