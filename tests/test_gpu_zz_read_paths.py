"""Routes of the device-planned read (scan_host.cc: enqueue_planned_read / download_planned) that the other GPU tests do not
reach: the borrowed read (lc_scan_read_borrowed), the selective byte-view get over host selections (lc_to_arrow_many,
one k_str_read_onepass launch) including its second round trip, and the launch and copy counts of the fused and
asynchronous reads. Every result is checked against Arrow's filter of the column."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from liquid_cache_b200 import BinaryExpr, Column, LiquidExpr, Literal
from tests.util import assert_arrays_equal

pytestmark = pytest.mark.gpu

HDR = 64  # sizeof(ScanPlanHdr) == sizeof(lc_read_header)


def _ge(v):
    return LiquidExpr.new_unchecked(BinaryExpr(Column("c", 0), ">=", Literal(v)))


def _value_bytes(a):
    return int(pc.sum(pc.binary_length(a)).as_py() or 0)


def _columns(cache, rng, n_batches, rows, scope):
    """int64 values in [0, 1000) and a Utf8 column of URLs, per batch; the handles keep the entries alive."""
    ints, strs, li, ls = [], [], [], []
    for b in range(n_batches):
        n = rows if b % 3 else rows - 37
        ints.append(pa.array(rng.integers(0, 1000, size=n), pa.int64()))
        strs.append(pa.array([f"http://h{int(rng.integers(0, 7))}.example/p/{int(rng.integers(0, 500))}" for _ in range(n)]))
        li.append(cache.transcode(ints[-1]))
        ls.append(cache.transcode(strs[-1], compressor_scope=scope))
    return ints, strs, li, ls


def _borrowed(cache, scan, h, typ):
    """(array over the scan's own device buffer copied to the host, d2h bytes the call moved), or (None, _)."""
    import torch

    d0 = cache.stats().d2h_bytes
    got = scan.read_torch_borrowed(h, torch.device("cuda", 0))
    d2h = cache.stats().d2h_bytes - d0
    if got is None:
        return None, d2h
    values, offsets, rows = got
    vb = pa.py_buffer(values.cpu().numpy().tobytes())
    if offsets is None:
        return pa.Array.from_buffers(typ, rows, [None, vb]), d2h
    return pa.Array.from_buffers(typ, rows, [None, pa.py_buffer(offsets.cpu().numpy().tobytes()), vb]), d2h


@pytest.mark.parametrize("kind", ["int64", "utf8"])
def test_borrowed_read_agrees_with_read(cache, kind):
    rng = np.random.default_rng(31 if kind == "int64" else 32)
    ints, strs, li, ls = _columns(cache, rng, 24, 4096, 8811 if kind == "int64" else 8815)
    hi = np.array([l.handle for l in li], dtype=np.uint64)
    hs = np.array([l.handle for l in ls], dtype=np.uint64)
    h, typ, col = (hi, pa.int64(), ints) if kind == "int64" else (hs, pa.string(), strs)
    is_str = kind == "utf8"

    def want(thr):
        return pa.concat_arrays([c.filter(pc.greater_equal(a, thr)) for a, c in zip(ints, col)])

    def fits(w, spec_rows, spec_bytes):  # the capacities scan_read_fused derives from the previous read
        return len(w) <= spec_rows + spec_rows // 2 + 4096 and (not is_str or _value_bytes(w) <= spec_bytes + spec_bytes // 2 + (64 << 10))

    with cache.scan([len(a) for a in ints]) as scan:
        assert _borrowed(cache, scan, h, typ)[0] is None  # no filter yet
        scan.filter(hi, _ge(500), pa.int64())
        assert _borrowed(cache, scan, h, typ)[0] is None  # filtered, but no read has taught the scan its sizes
        first = scan.read(h)
        assert_arrays_equal(first, want(500), "first read")
        spec_rows, spec_bytes = len(first), _value_bytes(first) if is_str else 0
        for thr in (600, 450):  # shrinks, then grows within the remembered capacities
            scan.reset()
            scan.filter(hi, _ge(thr), pa.int64())
            w = want(thr)
            assert fits(w, spec_rows, spec_bytes)
            got, d2h = _borrowed(cache, scan, h, typ)
            assert got is not None and d2h == HDR  # the header is all that crosses PCIe
            assert_arrays_equal(got, w, f"borrowed >= {thr}")
            again = scan.read(h)
            assert_arrays_equal(again, got, f"read >= {thr}")
            spec_rows, spec_bytes = len(again), _value_bytes(again) if is_str else 0
        # outgrows the capacities: refused, and the next read re-teaches the sizes
        scan.reset()
        scan.filter(hi, _ge(0), pa.int64())
        w = want(0)
        assert not fits(w, spec_rows, spec_bytes)
        assert _borrowed(cache, scan, h, typ)[0] is None
        assert_arrays_equal(scan.read(h), w, "read after the refusal")
        got, d2h = _borrowed(cache, scan, h, typ)
        assert got is not None and d2h == HDR
        assert_arrays_equal(got, w, "borrowed after re-learning")


@pytest.mark.parametrize("typ,rows,launches", [
    # 64 x 8192 rows: 16384 selection words, at most 1024 of them non-zero, so the selection travels as {word, value} pairs
    # and upload_selection scatters them (k_scatter_words) before the one k_str_read_onepass launch
    (pa.string(), 8192, 2),
    # 64 x 1000 rows: 2048 selection words, under the 4096 below which the words are copied as they are: one launch
    (pa.binary(), 1000, 1),
])
def test_selective_byte_view_get_over_host_selections(cache, typ, rows, launches):
    rng = np.random.default_rng(33 if typ == pa.string() else 34)
    n_entries = 64
    arrays, handles_keep = [], []
    for e in range(n_entries):
        # every 16th row is long (>= 300 bytes), the rest short
        vals = [(f"L{e}-{i}-" + "x" * 300) if i % 16 == 0 else f"s{int(rng.integers(0, 900))}" for i in range(rows)]
        arr = pa.array([v.encode() for v in vals], typ) if typ == pa.binary() else pa.array(vals, typ)
        arrays.append(arr)
        handles_keep.append(cache.transcode(arr, compressor_scope=8812 if typ == pa.string() else 8813))
    handles = np.array([l.handle for l in handles_keep], dtype=np.uint64)
    empty = {5, 40}  # entries without survivors

    def masks(long_rows):
        out = []
        for e in range(n_entries):
            m = np.zeros(rows, dtype=bool)
            if e not in empty:
                pool = np.arange(0, rows, 16) if long_rows else np.setdiff1d(np.arange(rows), np.arange(0, rows, 16))
                m[rng.choice(pool, size=int(rng.integers(1, 17)), replace=False)] = True
            out.append(m)
        return out

    def get(ms):
        sels = [np.packbits(m, bitorder="little") for m in ms]
        st0 = cache.stats()
        got = cache.to_arrow_many(handles, sels)
        st1 = cache.stats()
        want = pa.concat_arrays([a.filter(pa.array(m)) for a, m in zip(arrays, ms)])
        assert_arrays_equal(got, want, f"{typ} get")
        assert st1.kernel_launches - st0.kernel_launches == launches
        return want, st1.d2h_bytes - st0.d2h_bytes

    short, _ = get(masks(False))
    ratio = max(8.0, _value_bytes(short) / len(short))  # what the short read taught (onepass_bytes_per_row)
    ms = masks(True)
    want, d2h = get(ms)
    n_rows, n_bytes = len(want), _value_bytes(want)
    cap_bytes = sum(int(m.sum()) * max(len(v) for v in a.to_pylist()) for a, m in zip(arrays, ms))
    spec = min(cap_bytes, int(n_rows * ratio * 1.25) + 4096)
    assert n_bytes > spec  # larger than the speculative prefix: the values come again in a second round trip
    assert d2h == HDR + (n_rows + 1) * 4 + spec + n_bytes


def test_launch_and_copy_counts_of_the_fused_and_async_reads(cache):
    import torch

    rng = np.random.default_rng(35)
    n_batches = 64
    ints, strs, li, ls = _columns(cache, rng, n_batches, 4096, 8814)
    hi = np.array([l.handle for l in li], dtype=np.uint64)
    hs = np.array([l.handle for l in ls], dtype=np.uint64)
    dev = torch.device("cuda", 0)
    hdr = torch.zeros(HDR, dtype=torch.uint8, device=dev)
    values = torch.empty(16 << 20, dtype=torch.uint8, device=dev)
    offsets = torch.empty(300000, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()

    def async_read(h, rows_cap, want):
        cache.synchronize()
        st0 = cache.stats()
        assert scan.read_async(h, values.data_ptr(), values.numel(), offsets.data_ptr(), rows_cap, hdr.data_ptr())
        st1 = cache.stats()
        cache.synchronize()
        head = hdr.cpu().numpy()
        assert int(head[8:16].view(np.uint64)[0]) == len(want) and int(head[4:8].view(np.uint32)[0]) == 0
        return st1.kernel_launches - st0.kernel_launches, st1.h2d_bytes - st0.h2d_bytes, st1.d2h_bytes - st0.d2h_bytes

    with cache.scan([len(a) for a in ints]) as scan:
        thr = 999  # about 4 survivors per batch
        scan.filter(hi, _ge(thr), pa.int64())
        want_s = pa.concat_arrays([s.filter(pc.greater_equal(a, thr)) for a, s in zip(ints, strs)])
        assert 0 < len(want_s) <= 8 * n_batches
        # lc_scan_read_async. A first call builds the entry list (an upload); the counted call repeats it.
        for rows_cap, n_launch in ((16 * n_batches, 1),        # one-pass: k_str_read_onepass
                                   (16 * n_batches + 1, 5)):   # plan rows, sparse lengths, lengths, plan bytes, decode
            async_read(hs, rows_cap, want_s)
            assert async_read(hs, rows_cap, want_s) == (n_launch, 0, 0)
        want_i = pa.concat_arrays([a.filter(pc.greater_equal(a, thr)) for a in ints])
        async_read(hi, 4096, want_i)
        assert async_read(hi, 4096, want_i) == (2, 0, 0)  # plan rows, integer decode

        # lc_scan_read after a first read left <= 8 survivors per batch: the one-pass kernel
        assert_arrays_equal(scan.read(hs), want_s, "first read")
        k0 = cache.stats().kernel_launches
        assert_arrays_equal(scan.read(hs), want_s, "one-pass read")
        assert cache.stats().kernel_launches - k0 == 1
