"""`col [NOT] IN (list)` on the device (LC_OP_IN / LC_OP_NOT_IN), bit for bit against DataFusion's InListExpr semantics on
the decoded column: pyarrow.compute.is_in over the original values with nulls restored to null. The reference does not push
IN lists down (its LiquidExpr refuses them), so decode-then-compare IS its answer. Covers every integer physical type and
Date32 / Date64 / Timestamp, fields of <= 32 bits (k_int_bits) and wider ones (k_int_scan), nulls and selections, lists of
0 .. cap values, every byte-view type, all four entry points, refusals and launch counts."""
import ctypes as C
import datetime as dt
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from liquid_cache_b200 import _native as N
from liquid_cache_b200 import BinaryExpr, CacheExpression, Column, EntryID, InListExpr, LiquidExpr, Literal
from tests.util import assert_masks_equal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = N.IN_LIST_MAX_VALUES


def _expr(values, negated=False, col=None):
    return LiquidExpr.new_unchecked(InListExpr(col or Column("c"), tuple(Literal(v) for v in values), negated))


def _want(arr: pa.Array, values, negated, sel=None):
    """InListExpr on the decoded column: membership, negated for NOT IN, null rows null."""
    a = arr if sel is None else arr.filter(sel)
    if pa.types.is_dictionary(a.type):
        a = a.cast(a.type.value_type)
    vs = pa.array(list(values), type=a.type) if len(values) else pa.array([], type=a.type)
    m = pc.is_in(a, value_set=vs)
    if negated:
        m = pc.invert(m)
    return pc.if_else(pc.is_null(a), pa.scalar(None, pa.bool_()), m)


def _ints(rng, typ, n, lo, hi, null_p):
    vals = rng.integers(lo, hi, size=n, endpoint=True, dtype=np.int64 if lo < 0 else np.uint64)
    mask = rng.random(n) < null_p if null_p else None
    return pa.array(vals, type=pa.int64() if lo < 0 else pa.uint64(), mask=mask).cast(typ)


INT_TYPES = [(pa.int8(), -128, 127), (pa.uint8(), 0, 255), (pa.int16(), -30000, 30000), (pa.uint16(), 0, 65535),
             (pa.int32(), -(2**31), 2**31 - 1), (pa.uint32(), 0, 2**32 - 1), (pa.int64(), -(2**62), 2**62),
             (pa.uint64(), 0, 2**64 - 1)]


@pytest.mark.parametrize("typ,lo,hi", INT_TYPES, ids=lambda x: str(x))
@pytest.mark.parametrize("narrow", [True, False], ids=["w<=32", "wide"])
def test_integer_types_lists_nulls_selections(cache, typ, lo, hi, narrow):
    rng = np.random.default_rng(typ.bit_width * 7 + narrow)
    base = max(lo, -500) if narrow else lo  # narrow: a window of at most 1001 values (W <= 10); wide: the whole type
    top = min(hi, base + 1000) if narrow else hi
    arr_full = _ints(rng, typ, 8192 * 3 + 77, base, top, 0.0)
    arr_null = _ints(rng, typ, 8192 * 2 + 5, base, top, 0.1)
    sel = pa.array(rng.random(len(arr_null)) < 0.6)
    present = [v for v in arr_full.to_pylist()[:4000]]
    for arr, s in ((arr_full, None), (arr_null, None), (arr_null, sel)):
        g = cache.transcode(arr)
        for k in (0, 1, 2, 8, 64, CAP):
            vals = [int(x) for x in rng.choice(present, size=k)] if k else []
            if k >= 8:  # values outside the data and the type's extremes
                vals[:3] = [lo, hi, base - 1 if base - 1 >= lo else hi]
            if k == 2:
                vals = [vals[0], vals[0] + 1]  # a consecutive run
            for neg in (False, True):
                got = g.try_eval_predicate(_expr(vals, neg), s)
                assert_masks_equal(got, _want(arr, vals, neg, s), f"{typ} narrow={narrow} k={k} neg={neg} sel={s is not None}")


def test_negative_literals_and_above_i64(cache):
    arr = pa.array([2**63 + 1, 5, 2**64 - 1, None, 0, 2**63 + 1], pa.uint64())
    g = cache.transcode(arr)
    for vals in ([2**63 + 1, 0], [2**64 - 1], [-1, 5], [-5]):
        for neg in (False, True):
            if any(v < 0 for v in vals) and any(v > 2**63 for v in vals):
                continue
            assert_masks_equal(g.try_eval_predicate(_expr(vals, neg), None), _want(arr, [v for v in vals if v >= 0], neg), str(vals))
    arr = pa.array([-3, -2, None, 7, -128], pa.int8())
    g = cache.transcode(arr)
    for vals in ([-3, -128, 1000], [-2, -1, 7], [1000, -1000], [2**63 + 9, 127]):
        want = _want(arr, [v for v in vals if -128 <= v <= 127], False)
        assert_masks_equal(g.try_eval_predicate(_expr(vals), None), want, str(vals))


@pytest.mark.parametrize("typ", [pa.date32(), pa.date64(), pa.timestamp("us"), pa.timestamp("ms")], ids=str)
def test_dates_and_timestamps(cache, typ):
    rng = np.random.default_rng(3)
    if pa.types.is_date32(typ):
        raw = rng.integers(15000, 16000, size=9000)
        vals = [dt.date(1970, 1, 1) + dt.timedelta(days=int(d)) for d in rng.choice(raw, 20)]
    elif pa.types.is_date64(typ):
        raw = rng.integers(15000, 16000, size=9000) * 86_400_000
        vals = [dt.date(1970, 1, 1) + dt.timedelta(days=int(d) // 86_400_000) for d in rng.choice(raw, 20)]
    else:
        raw = rng.integers(10**12, 10**12 + 10**7, size=9000)
        vals = [int(x) for x in rng.choice(raw, 20)]
    if pa.types.is_date32(typ):
        phys = pa.array(raw.astype(np.int32), pa.int32())
        ints = [(v - dt.date(1970, 1, 1)).days for v in vals]
    else:
        phys = pa.array(raw, pa.int64())
        ints = [(v - dt.date(1970, 1, 1)).days * 86_400_000 for v in vals] if pa.types.is_date64(typ) else vals
    arr = phys.cast(typ)
    g = cache.transcode(arr)
    got = g.try_eval_predicate(_expr(vals), None)
    want = pc.is_in(phys, value_set=pa.array(ints, phys.type))
    assert_masks_equal(got, want, str(typ))


def _strings(rng, n, null_p=0.0):
    long = "x" * 300
    pool = ["", "a", "MAIL", "SHIP", "AIR", "AIR REG", "TRUCK", "http://example.org/page/1", "http://example.org/page/2",
            "http://example.org/page/22", long, long + "y", "SM CASE", "SM BOX", "LG PACK", "prefix-only"]
    idx = rng.integers(0, len(pool), size=n)
    mask = rng.random(n) < null_p if null_p else None
    return pa.array([pool[i] for i in idx], pa.string(), mask=mask), pool


NEEDLE_LISTS = [[], ["MAIL"], ["MAIL", "SHIP"], ["AIR", "AIR REG"], ["http://example.org/page/2", "http://example.org/page/22"],
                ["x" * 300, "nope", "x" * 301], [""], ["absent", "also absent", "http://example.org/page/3"]]


@pytest.mark.parametrize("kind", ["utf8", "binary", "utf8_view", "binary_view", "dict"])
def test_byte_view_types(cache, kind):
    rng = np.random.default_rng(11)
    arr, pool = _strings(rng, 8192 * 2 + 9, 0.1)
    if kind == "binary":
        arr = arr.cast(pa.binary())
    elif kind == "utf8_view":
        arr = arr.cast(pa.string_view())
    elif kind == "binary_view":
        arr = arr.cast(pa.binary_view())
    elif kind == "dict":
        arr = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(pool), size=5000), pa.uint16()), pa.array(pool))
    sel = pa.array(rng.random(len(arr)) < 0.5)
    for hint in (None, CacheExpression.SubstringSearch):
        g = cache.transcode(arr, hint=hint)
        for vals in NEEDLE_LISTS + [pool, [p + "z" for p in pool] * 16]:
            enc = [v.encode() for v in vals] if kind in ("binary", "binary_view") else vals
            for neg in (False, True):
                for s in (None, sel):
                    got = g.try_eval_predicate(_expr(enc, neg), s)
                    want = _want(arr.cast(pa.string()) if kind != "dict" else arr, vals, neg, s)
                    assert_masks_equal(got, want, f"{kind} hint={hint} {vals[:3]} neg={neg} sel={s is not None}")


def test_shared_prefix_longer_than_needles(cache):
    arr = pa.array(["http://host/a", "http://host/bb", None, "http://host/a", "http://host/abcdefghijk"] * 50)
    g = cache.transcode(arr)
    for vals in (["http", "http://host/a"], ["http://host/abcdefghijk", "http://host/abcdefghijj"], ["http://host/"]):
        for neg in (False, True):
            assert_masks_equal(g.try_eval_predicate(_expr(vals, neg), None), _want(arr, vals, neg), str(vals))


def test_lqda_round_trip(cache):
    rng = np.random.default_rng(5)
    arr, pool = _strings(rng, 6000)
    scope = 0x77
    g = cache.transcode(arr, compressor_scope=scope)
    back = cache.read_from_bytes(g.to_bytes(), compressor_scope=scope)
    for vals in (["MAIL", "SHIP"], ["x" * 300, "TRUCK"]):
        assert_masks_equal(back.try_eval_predicate(_expr(vals), None), _want(arr, vals, False), "lqda strings")
    ia = _ints(rng, pa.int32(), 5000, -100, 100, 0.05)
    gi = cache.read_from_bytes(cache.transcode(ia).to_bytes())
    assert_masks_equal(gi.try_eval_predicate(_expr([-5, 0, 7, 99]), None), _want(ia, [-5, 0, 7, 99], False), "lqda ints")


def test_entry_points_and_scan(cache):
    rng = np.random.default_rng(8)
    n_b = 6
    ints = [_ints(rng, pa.int32(), 8192, 0, 50, 0.05) for _ in range(n_b)]
    wide = [_ints(rng, pa.int64(), 8192, -(2**50), 2**50, 0.0) for _ in range(n_b)]
    strs = [_strings(rng, 8192, 0.05)[0] for _ in range(n_b)]
    ids_i = [EntryID(9000 + i) for i in range(n_b)]
    ids_w = [EntryID(9100 + i) for i in range(n_b)]
    ids_s = [EntryID(9200 + i) for i in range(n_b)]
    cache.insert_many(ids_i, ints)
    cache.insert_many(ids_w, wide)
    cache.insert_many(ids_s, strs)
    # lc_cache_eval_predicate
    got = cache.eval_predicate(ids_i[0], _expr([3, 7, 11])).read()
    assert_masks_equal(got, _want(ints[0], [3, 7, 11], False), "cache eval")
    # lc_eval_predicate_many
    hi = cache.handles(ids_i)
    rows = np.array([len(a) for a in ints], dtype=np.uint64)
    vals, valid, offs, out_len, nulls, _t = cache.eval_predicate_many(hi, rows, _expr([1, 2, 3, 40], True), pa.int32())
    for i in range(n_b):
        nb = (int(out_len[i]) + 7) // 8
        bits = np.unpackbits(vals[offs[i]:offs[i] + nb], bitorder="little")[: int(out_len[i])].astype(bool)
        vb = np.unpackbits(valid[offs[i]:offs[i] + nb], bitorder="little")[: int(out_len[i])].astype(bool)
        got = pa.array(bits, mask=~vb)
        assert_masks_equal(got, _want(ints[i], [1, 2, 3, 40], True), f"many {i}")
    # lc_scan_filter composed with other conjuncts, then lc_scan_read
    wl = [int(x) for x in rng.choice(pa.concat_arrays(wide).to_numpy(), 64)]
    with cache.scan([8192] * n_b) as sc:
        sc.filter(hi, LiquidExpr.new_unchecked(BinaryExpr(Column("c"), ">", Literal(5))), pa.int32())
        sc.filter(cache.handles(ids_s), _expr(["MAIL", "SHIP", "x" * 300]), pa.string())
        sc.filter(hi, _expr([6, 7, 8, 20, 33]), pa.int32())
        got = sc.read(cache.handles(ids_s))
        want = []
        for i in range(n_b):
            m = pc.and_(pc.and_(pc.greater(ints[i], 5), pc.is_in(strs[i], value_set=pa.array(["MAIL", "SHIP", "x" * 300]))),
                        pc.is_in(ints[i], value_set=pa.array([6, 7, 8, 20, 33], pa.int32())))
            want.append(strs[i].filter(m.fill_null(False)))
        assert got.to_pylist() == pa.concat_arrays(want).to_pylist()
        sc.reset()
        sc.filter(cache.handles(ids_w), _expr(wl, True), pa.int64())
        counts, total = sc.counts()
        want_w = sum(int(pc.sum(pc.invert(pc.is_in(a, value_set=pa.array(wl, pa.int64())))).as_py()) for a in wide)
        assert total == want_w


def test_refusals_leave_the_selection_unchanged(cache):
    rng = np.random.default_rng(9)
    fl = pa.array(rng.random(8192))
    dec = pa.array([1, 2, 3] * 100, pa.int64()).cast(pa.decimal128(21, 2))
    ints = _ints(rng, pa.int32(), 8192, 0, 1000, 0.0)
    for e, arr in ((EntryID(9300), fl), (EntryID(9301), dec), (EntryID(9302), ints)):
        cache.insert(e, arr).run()
    with cache.scan([8192]) as sc:
        sc.filter(cache.handles([EntryID(9302)]), LiquidExpr.new_unchecked(BinaryExpr(Column("c"), "<", Literal(500))), pa.int32())
        before = sc.store_selections().copy()
        with pytest.raises(N.UnsupportedExpr):
            sc.filter(cache.handles([EntryID(9302)]), _expr(list(range(CAP + 1))), pa.int32())
        p = N.Predicate()
        p.op, p.lit_kind, p.lit_len = N.OP_IN, N.LIT_I64, 1
        one = np.array([1], dtype="<i8").tobytes()
        p._keepalive = one
        p.lit_bytes = one
        with pytest.raises(N.UnsupportedExpr):
            sc.filter_native(cache.handles([EntryID(9300)]), p)  # float entry
        assert np.array_equal(sc.store_selections(), before)
    with pytest.raises(N.UnsupportedExpr):
        cache.transcode(fl).try_eval_predicate(_expr([0.5]), None)
    g = cache.transcode(dec)
    with pytest.raises(N.UnsupportedExpr):
        N.check(N.lib().lc_eval_predicate(cache._ctx, g._h, C.byref(p), None, 0, np.zeros(64, np.uint8).ctypes.data, None,
                                          C.byref(C.c_uint64()), C.byref(C.c_uint64())))
    sa = pa.array(["a", "b"] * 100)
    with pytest.raises(N.UnsupportedExpr):
        cache.transcode(sa).try_eval_predicate(_expr(["v%d" % i for i in range(CAP + 1)]), None)
    with pytest.raises(N.UnsupportedExpr):
        cache.transcode(sa).try_eval_predicate(_expr(["y" * 200] * 100), None)  # 20000 value bytes > the byte cap
    # a malformed byte list: offsets that decrease
    bad = np.array([0, 5, 2], dtype="<i4").tobytes() + b"abcde"
    q = N.Predicate()
    q.op, q.lit_kind, q.lit_len = N.OP_IN, N.LIT_BYTES, 2
    q._keepalive = bad
    q.lit_bytes = bad
    gs = cache.transcode(sa)
    rc = N.lib().lc_eval_predicate(cache._ctx, gs._h, C.byref(q), None, 0, np.zeros(64, np.uint8).ctypes.data, None,
                                   C.byref(C.c_uint64()), C.byref(C.c_uint64()))
    assert rc == N.LC_ERR_INVALID


def test_squeezed_entries_refuse(cache):
    from liquid_cache_b200.cache import GpuSqueezedArray  # noqa: F401

    rng = np.random.default_rng(10)
    arr = _ints(rng, pa.int64(), 8192, 0, 2**40, 0.0)
    g = cache.transcode(arr)
    try:
        sq = g.squeeze("clamp", CacheExpression.PredicateColumn)
    except Exception:
        pytest.skip("this build's squeeze front door has another shape")
    if sq is None:
        pytest.skip("entry did not squeeze")
    sq_arr = sq[0] if isinstance(sq, tuple) else sq
    with pytest.raises(N.UnsupportedExpr):
        sq_arr.try_eval_predicate(_expr([1, 2]), None)


def test_in_launches_as_many_kernels_as_eq(cache):
    rng = np.random.default_rng(12)
    ints = [_ints(rng, pa.int32(), 8192, 0, 1000, 0.0) for _ in range(4)]
    ids = [EntryID(9400 + i) for i in range(4)]
    cache.insert_many(ids, ints)
    h = cache.handles(ids)
    strs = [_strings(rng, 8192)[0] for _ in range(4)]
    sids = [EntryID(9500 + i) for i in range(4)]
    cache.insert_many(sids, strs)
    hs = cache.handles(sids)
    for handles, typ, eq, lst in ((h, pa.int32(), 17, [17, 300, 999]), (hs, pa.string(), "MAIL", ["MAIL", "SHIP", "AIR"])):
        with cache.scan([8192] * 4) as sc:
            sc.filter(handles, LiquidExpr.new_unchecked(BinaryExpr(Column("c"), "=", Literal(eq))), typ)  # warm the entry list
            k0 = cache.stats().kernel_launches
            sc.filter(handles, LiquidExpr.new_unchecked(BinaryExpr(Column("c"), "=", Literal(eq))), typ)
            k1 = cache.stats().kernel_launches
            sc.filter(handles, _expr(lst), typ)
            k2 = cache.stats().kernel_launches
        assert k2 - k1 == k1 - k0, (str(typ), k1 - k0, k2 - k1)


def test_cpp_mirror_answers_in_lists():
    lib_dir = os.path.join(ROOT, "liquid_cache_b200", "lib")
    exe = os.path.join(ROOT, "build", "tests", "in_list_mirror")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT}", os.path.join(ROOT, "tests", "cpp", "in_list_mirror.cc"),
                        "-o", exe, f"-L{lib_dir}", "-llc_gpu", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "0 wrong answers" in r.stdout, (r.returncode, r.stdout, r.stderr)
