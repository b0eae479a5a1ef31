"""The sweep's device IN-list variant of q40 (bench_sweep.py: the IN conjunct as an `lc_scan_filter` with LC_OP_IN, next to
the reference-shaped host path) over a pyarrow test double that evaluates InListExpr the way the native scan does. No GPU
needed: this checks the harness — the conjunct lowers through LiquidExpr.to_native, both variants' survivor counts equal
Arrow's, and the second total replaces q40's host time with the device one."""
import time

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

import bench_sweep as S
from tests import fake_cache as F


class _InListScan(F.FakeScanWords):
    """The bulk-selection double plus what the native scan has and the double lacks: InListExpr filters (`filter_native` is
    how the sweep recognises such a scan)."""

    def filter(self, handles, expr, column_type):
        from liquid_cache_b200 import InListExpr

        e = expr.physical_expr()
        if not isinstance(e, InListExpr):
            return super().filter(handles, expr, column_type)
        expr.to_native(column_type)  # the lowering the real call performs
        for b, h in enumerate(handles):
            arr = self.cache.store[int(h)]
            m = pc.is_in(arr, value_set=pa.array([it.value for it in e.list], arr.type))
            m = pc.invert(m) if e.negated else m
            self.sel[b] &= np.asarray(m.fill_null(False).to_numpy(zero_copy_only=False), dtype=bool)

    def filter_native(self, handles, pred):
        raise NotImplementedError


class _InListCache(F.FakeCache):
    def scan(self, rows):
        return _InListScan(self, rows)


def _timer():
    t = [0.0]

    def start():
        t[0] = time.perf_counter()

    return start, (lambda: (time.perf_counter() - t[0]) * 1e3)


def test_q40_runs_both_ways_and_both_match_arrow():
    res = S.run_sweep(_InListCache(bulk_selections=True), rows=8192 * 24, steps=1, warmup=1, timer=_timer, check_batches=24)
    assert res["all_counts_match_arrow"]
    by_q = {r["q"]: r for r in res["queries"]}
    dev = by_q[40]["device_in_list"]
    assert dev["counts_match_arrow"] and dev["rows_out"] == by_q[40]["rows_out"]
    assert [q for q, r in by_q.items() if "device_in_list" in r] == [40]  # the only query with an IN conjunct
    want = res["sweep_ms"] - by_q[40]["ms"] + dev["ms"]
    assert abs(res["sweep_ms_device_in_list"] - want) < 1e-9


def test_the_plain_double_keeps_the_host_path_only():
    res = S.run_sweep(F.FakeCache(bulk_selections=True), rows=8192 * 8, steps=1, warmup=1, timer=_timer, check_batches=8)
    assert res["all_counts_match_arrow"]
    assert not any("device_in_list" in r for r in res["queries"])
    assert res["sweep_ms_device_in_list"] == res["sweep_ms"]
