"""Every kernel of the low- and mid-cardinality aggregate paths (agg_tile.cu, agg_priv.cu) and of the generic table
(agg.cu), forced by its shape or knob, checked against an exact reference AND against the kernel trace: the
dispatchers fall back silently (FASTREG -> FAST, PRIV -> WPRIV -> MID, any of them -> the global row path), and every
fall-back computes the same answer, so without the trace a test written for one kernel could be testing another.

Integer sums, counts and integer AVG are bit-exact (sums as Python ints, AVG as long double(sum) / count like the
library's finalize); MIN / MAX bit-exact; double sums within 1e-9 relative.  Inputs sit on the edges of the fast paths:
values on both sides of the 2^40 limit of the 64-bit per-thread partials, INT64 / UINT64 extremes, NULLs that only
arrive in a later batch, keys first seen after the adaptation probe."""
import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran, kernel_trace, ran
from oracle import port as P
from test_gpu_kernel_paths import _download_raw

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of agg_tile.cu, agg_priv.cu, agg.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "agg_fastreg_kernel": ["test_ubigint_sum_near_2_64", "test_fastreg_kernels", "test_fastreg_row_counts",
                           "test_generic_table_growth_and_replay"],
    "agg_fast_kernel": ["test_fast_kernel_shapes", "test_fast_partial_overflow", "test_minmax_type_limits"],
    "agg_priv_kernel": ["test_ubigint_sum_near_2_64", "test_priv_kernels", "test_priv_direct_edges"],
    "agg_wpriv_kernel": ["test_ubigint_sum_near_2_64", "test_priv_kernels", "test_priv_direct_edges"],
    "agg_mid_kernel": ["test_mid_kernel", "test_mid_spill", "test_minmax_type_limits",
                       "test_more_columns_than_a_tile_stage_takes"],
    "agg_mid2_kernel": ["test_ubigint_sum_near_2_64", "test_mid2_kernel", "test_mid2_periodic_flushes"],
    "agg_list_keys_kernel": ["test_priv_kernels"],
    "agg_init_kernel": ["test_generic_table_growth_and_replay"],
    "agg_sink_kernel": ["test_generic_table_growth_and_replay", "test_mid_not_for_long_keys",
                        "test_more_columns_than_a_tile_stage_takes"],
    "agg_rehash_kernel": ["test_generic_table_growth_and_replay"],
    "agg_fix_cnt_kernel": ["test_validity_arrives_later"],
    "agg_finalize_kernel": ["test_generic_table_growth_and_replay"],
    "agg_export_kernel": ["test_export_combine_states"],
    "agg_combine_kernel": ["test_export_combine_states"],
    "agg_export_packed_kernel": ["test_packed_three_ranks"],
    "agg_packed_header_kernel": ["test_packed_three_ranks"],
    "agg_combine_packed_kernel": ["test_packed_three_ranks", "test_packed_overflow_is_reported"],
    "fill_u64_kernel3": ["test_generic_table_growth_and_replay"],
}
# kernels of those files that no test here has to reach, with the reason
KERNEL_EXCLUDED = {}

PROBE = 1 << 18  # rows of the adaptation probe chunk (b200_agg_sink)
FUNC = {"count_star": capi.AGG_COUNT_STAR, "count": capi.AGG_COUNT, "sum": capi.AGG_SUM,
        "sum_no_overflow": capi.AGG_SUM_NO_OVERFLOW, "min": capi.AGG_MIN, "max": capi.AGG_MAX, "avg": capi.AGG_AVG}
SIGNED_EDGES = [-2 ** 40 - 1, -2 ** 40, 2 ** 40 - 1, 2 ** 40, -2 ** 63, 2 ** 63 - 1]
UNSIGNED_EDGES = [2 ** 40 - 1, 2 ** 40, 2 ** 63, 2 ** 64 - 2 ** 40, 2 ** 64 - 1]
NOT_LOW_CARD = ["agg_fastreg_kernel", "agg_fast_kernel", "agg_priv_kernel", "agg_wpriv_kernel", "agg_mid_kernel",
                "agg_mid2_kernel"]


def traced_window(fn, always):
    """-> (fn(), kernel names).  The profiler occasionally drops a window's kernel records, whole or in part; a window
    that misses one of the kernels `always` (kernels fn launches on every call, e.g. agg_init_kernel: every aggregate
    initialises its table) says nothing about the dispatcher, so fn, which must be repeatable, runs again in a fresh
    window, up to three windows.  Three windows without a kernel are an error; after three incomplete ones the last
    is returned for the caller's assertions to report."""
    for attempt in range(3):
        with kernel_trace() as names:
            result = fn()
        if names and all(ran(names, k) for k in always):
            return result, names
    assert names, "torch.profiler recorded no CUDA kernel in three windows that launched kernels"
    return result, names


# ------------------------------------------------------------------ exact references
def exact_group_sums(gid, ng, v, valid=None):
    """per-group sums of integers as Python ints: 16-bit limbs summed by bincount (a limb sum stays below 2^53 for any
    row count below 2^37, so the float64 accumulation is exact), recombined with Python ints"""
    v = np.asarray(v)
    u = v.astype(np.int64).view(np.uint64) if v.dtype.kind == "i" else v.astype(np.uint64)
    w = None if valid is None else valid.astype(np.float64)
    total = np.zeros(ng, dtype=object)
    for k in range(4):
        limb = (u >> np.uint64(16 * k)) & np.uint64(0xFFFF)
        x = limb.astype(np.float64)
        if k == 3 and v.dtype.kind == "i":
            x = np.where(limb >= 0x8000, x - 65536.0, x)  # the top limb of a signed value carries the sign
        s = np.bincount(gid, weights=x if w is None else x * w, minlength=ng)
        total = total + s.astype(np.int64).astype(object) * (1 << (16 * k))
    return total


def ld_avg(s, c):
    """integer AVG as the library finalizes it: the 128-bit sum converted to long double (high word * 2^64 + low
    word, each exact), divided by the count in long double, rounded to double"""
    if c == 0:
        return None
    neg = s < 0
    a = -s if neg else s
    hi, lo = divmod(a, 1 << 64)
    v = np.longdouble(np.uint64(hi)) * (np.longdouble(2.0) ** 64) + np.longdouble(np.uint64(lo))
    return float((-v if neg else v) / np.longdouble(c))


def canon(x):
    """a key value as the finalized batch reports it: Python int, or the canonical bit pattern of a double"""
    if isinstance(x, (float, np.floating)):
        x = float(x)
        if x == 0.0:
            return 0
        if np.isnan(x):
            return 0x7FF8000000000000
        return int(np.array([x]).view(np.uint64)[0])
    return int(x)


def group_minmax(gid, ng, v, valid, func):
    """MIN / MAX of integers per group (groups without a valid value: None)"""
    v = np.asarray(v)
    sel = np.ones(len(v), dtype=bool) if valid is None else valid
    info = np.iinfo(v.dtype)
    out = np.full(ng, info.max if func == "min" else info.min, dtype=v.dtype)
    (np.minimum if func == "min" else np.maximum).at(out, gid[sel], v[sel])
    has = np.bincount(gid[sel], minlength=ng) > 0
    return [int(out[g]) if has[g] else None for g in range(ng)]


def reference(keys, gid, ng, inputs, aggs):
    """keys: [(values, valid|None)] per row; gid: group index of every row (rows of one group share one canonical key);
    inputs: [(values, valid|None)]; aggs: [(func, input index | -1)].  -> {key tuple: [result per aggregate]}"""
    n = len(gid)
    rows = np.bincount(gid, minlength=ng)
    first = np.full(ng, -1, dtype=np.int64)
    first[gid[::-1]] = np.arange(n - 1, -1, -1)
    cache = {}
    cols = []
    for f, i in aggs:
        if f == "count_star":
            cols.append([int(r) for r in rows])
            continue
        v, valid = inputs[i]
        cnt = rows if valid is None else np.bincount(gid, weights=valid, minlength=ng).astype(np.int64)
        if f == "count":
            cols.append([int(c) for c in cnt])
        elif np.asarray(v).dtype.kind == "f":
            w = np.where(valid, v, 0.0) if valid is not None else v
            s = np.bincount(gid, weights=w, minlength=ng)
            if f == "sum":
                cols.append([float(s[g]) if cnt[g] else None for g in range(ng)])
            elif f == "avg":
                cols.append([float(s[g]) / int(cnt[g]) if cnt[g] else None for g in range(ng)])
            else:
                raise ValueError(f)  # double MIN / MAX: oracle.port.group_by (NaN ordering)
        elif f in ("min", "max"):
            cols.append(group_minmax(gid, ng, v, valid, f))
        else:
            if i not in cache:
                cache[i] = exact_group_sums(gid, ng, v, valid)
            s = cache[i]
            if f == "sum":
                cols.append([int(s[g]) if cnt[g] else None for g in range(ng)])
            elif f == "sum_no_overflow":
                cols.append([(int(s[g]) + 2 ** 63) % 2 ** 64 - 2 ** 63 if cnt[g] else None for g in range(ng)])
            elif f == "avg":
                cols.append([ld_avg(int(s[g]), int(cnt[g])) for g in range(ng)])
            else:
                raise ValueError(f)
    out = {}
    for g in np.nonzero(rows)[0]:
        r = first[g]
        key = tuple(canon(k[r]) if kv is None or kv[r] else None for k, kv in keys)
        assert key not in out, f"groups {g} and another share the key {key}: the test data is wrong"
        out[key] = [c[g] for c in cols]
    return out


def fetch_groups(batch, nkeys, naggs):
    """finalize() output -> {key tuple: [result per aggregate]}, values as Python scalars, NULL as None"""
    res = _download_raw(batch)
    out = {}
    for g in range(batch.nrows):
        key = tuple(canon(res[j][0][g]) if res[j][1][g] else None for j in range(nkeys))
        assert key not in out, f"duplicate group {key} in the output"
        vals = []
        for a in range(naggs):
            v, ok = res[nkeys + a]
            x = v[g]
            vals.append((x if isinstance(x, int) else x.item()) if ok[g] else None)
        out[key] = vals
    return out


def assert_same(got, exp, aggs, inputs):
    assert len(got) == len(exp), (len(got), len(exp))
    assert set(got) == set(exp), sorted(set(got) ^ set(exp))[:10]
    for k, e in exp.items():
        for (f, i), gv, ev in zip(aggs, got[k], e):
            isf = i >= 0 and np.asarray(inputs[i][0]).dtype.kind == "f"
            if ev is None or gv is None:
                assert gv is None and ev is None, (k, f, i, gv, ev)
            elif isinstance(ev, float) and np.isnan(ev):
                assert np.isnan(gv), (k, f, i, gv)
            elif isf and f in ("sum", "avg"):
                assert gv == pytest.approx(ev, rel=1e-9, abs=1e-12), (k, f, i, gv, ev)
            else:
                assert gv == ev, (k, f, i, gv, ev)  # bit-exact, AVG included


def descs_of(aggs, inputs):
    return [(FUNC[f], capi.TYPE_OF_DTYPE[np.asarray(inputs[i][0]).dtype] if i >= 0 else capi.INT64, i)
            for f, i in aggs]


def sink_all(ctx, agg, keys, inputs, bounds, masked=None):
    """sink rows in batches [bounds[b], bounds[b+1]); masked[b][i]: pass input i's validity in batch b (default: when
    it has one).  A batch sent without a mask must have no NULLs in it."""
    for b, (lo, hi) in enumerate(zip(bounds[:-1], bounds[1:])):
        vs = [ops.Vector.flat(k[lo:hi], None if kv is None else kv[lo:hi]) for k, kv in keys]
        for i, (v, valid) in enumerate(inputs):
            use = valid is not None and (masked is None or masked[b][i])
            if valid is not None and not use:
                assert valid[lo:hi].all(), "a batch without a validity mask must not hold NULLs"
            vs.append(ops.Vector.flat(v[lo:hi], valid[lo:hi] if use else None))
        agg.sink(ops.Batch.upload(ctx, vs, int(hi - lo)), list(range(len(keys))),
                 list(range(len(keys), len(keys) + len(inputs))))


def agg_run(ctx, keys, gid, ng, inputs, aggs, bounds=None, masked=None, expected_groups=0, exp=None):
    """sink + finalize inside the kernel trace, check against the exact reference (or `exp`); -> kernel names"""
    n = len(gid)
    bounds = [0, n] if bounds is None else bounds
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]

    def run():
        agg = ops.HashAggregate(ctx, key_types, descs_of(aggs, inputs), expected_groups)
        sink_all(ctx, agg, keys, inputs, bounds, masked)
        out = fetch_groups(agg.finalize(), len(keys), len(aggs))
        agg.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel"])   # (every aggregate initialises its table)
    assert_same(got, reference(keys, gid, ng, inputs, aggs) if exp is None else exp, aggs, inputs)
    return names


def planted(rng, dtype, n, lo, hi, count=40):
    """random values in [lo, hi) with the fast paths' edge values planted at random rows"""
    v = rng.integers(lo, hi, size=n, dtype=dtype)
    if n:
        edges = SIGNED_EDGES if np.dtype(dtype).kind == "i" else UNSIGNED_EDGES
        for e in edges:
            v[rng.integers(0, n, size=min(count, n))] = e
    return v


def sum_inputs(rng, nsum, n):
    """nsum 8-byte columns, INT64 and UINT64 alternately, inside the fast range with the edge values planted"""
    return [(planted(rng, np.int64, n, -2 ** 39, 2 ** 39) if j % 2 == 0 else
             planted(rng, np.uint64, n, 0, 2 ** 40), None) for j in range(nsum)]


def sum_aggs(nsum):
    """SUM of every input; AVG, SUM_NO_OVERFLOW and COUNT of input 0; COUNT(*)"""
    return [("sum", j) for j in range(nsum)] + [("avg", 0), ("sum_no_overflow", 0), ("count", 0), ("count_star", -1)]


# ------------------------------------------------------------------ key forms
def key_columns(form, gid, ng):
    """group index -> key columns of one of the register path's key shapes.  kw1: 1..4 one-byte keys (UTINYINT and
    TINYINT, negative values included); kw4: one INTEGER (negative values included); kw0: SMALLINT + TINYINT or
    USMALLINT + UINTEGER (generic key descriptors).  Every group gets a distinct key."""
    g = gid.astype(np.int64)
    if form.startswith("kw1"):
        nk = int(form[-1])
        cols, rest = [], g.copy()
        for j in range(nk):
            base = ng if j == nk - 1 else 3
            digit = rest % base if j < nk - 1 else rest
            rest = rest // base
            cols.append(((digit - 2).astype(np.int8), None) if j % 2 else (digit.astype(np.uint8), None))
        return cols
    if form == "kw4":
        return [(((g - ng // 2) * 1_000_003).astype(np.int32), None)]
    # (kw0: few distinct values per column, so that the PRIV path's direct slot tables - the cross product of the
    # columns' values - stay within its slots)
    if form == "kw0s":
        return [(((g >> 1) + 30000).astype(np.int16), None), (((g & 1) * 3 - 1).astype(np.int8), None)]
    if form == "kw0u":
        return [((g // 5 + 60000).astype(np.uint16), None), ((g % 5 * 3 + 2 ** 31).astype(np.uint32), None)]
    raise ValueError(form)


def fastreg_kw(form):
    return 1 if form.startswith("kw1") else 4 if form == "kw4" else 0


def fastreg_threads(slots, nsum):
    """consumer threads of agg_fastreg_kernel<NSUM, SLOTS, THREADS, KW>: fewer as the register accumulators grow"""
    return 224 if slots * nsum <= 20 else 192 if slots * nsum <= 32 else 160


# ------------------------------------------------------------------ the UBIGINT sum bug
@pytest.mark.parametrize("path", ["fastreg", "priv", "wpriv", "mid2"])
def test_ubigint_sum_near_2_64(ctx, monkeypatch, path):
    """SUM / AVG over UBIGINT values in [2^64 - 2^40, 2^64).  The fast paths send a value to the exact global path when
    it is too large for their 64-bit per-thread partials; the test used to be the signed one, (x + 2^40) >> 41, and
    for such an unsigned x the addition wrapped, so the value stayed in a partial that the reduction widens as signed:
    SUM(UBIGINT) over {2^64 - 1, 1} returned 0 instead of 2^64.  MID2's limb range test had the same wrap."""
    rng = np.random.default_rng(1)
    if path == "fastreg":
        ng, n = 3, 4000
    elif path == "mid2":
        ng, n = 3, 300_000
        monkeypatch.setenv("B200_AGG_MID2", "704")
    else:
        ng, n = 35, 600_000
        monkeypatch.setenv("B200_AGG_WPRIV" if path == "wpriv" else "B200_AGG_NO_WPRIV", "1")
    gid = rng.integers(0, ng, size=n)
    u = rng.integers(0, 2 ** 40, size=n, dtype=np.uint64)
    u[gid == 0] = np.uint64(1)
    rows0 = np.nonzero(gid == 0)[0]
    u[rows0[: len(rows0) // 2]] = np.uint64(2 ** 64 - 1)        # group 0: about half 2^64 - 1, half 1
    for e in UNSIGNED_EDGES:
        u[rng.integers(0, n, size=30)] = np.uint64(e)
    s = rng.integers(-2 ** 39, 2 ** 39, size=n, dtype=np.int64)
    inputs = [(u, None), (s, None)]
    aggs = [("sum", 0), ("avg", 0), ("sum", 1), ("count_star", -1)]
    if path == "mid2":
        keys = [(gid.astype(np.int64) * 2 ** 40 - 5, None)]  # 8-byte key: the shared-memory table (MID) from the first row
    else:
        keys = [((gid // 5).astype(np.uint8), None), ((gid % 5).astype(np.uint8), None)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    if path == "fastreg":
        assert_ran(names, "agg_fastreg_kernel<2, 4, 224, 1>")
        assert_not_ran(names, "agg_fast_kernel", "agg_mid_kernel")
    elif path == "priv":
        assert_ran(names, "agg_priv_kernel<2, 2>")
        assert_not_ran(names, "agg_wpriv_kernel", "agg_mid_kernel")
    elif path == "wpriv":
        assert_ran(names, "agg_wpriv_kernel<2>")
        assert_not_ran(names, "agg_priv_kernel", "agg_mid_kernel")
    else:
        assert_ran(names, "agg_mid2_kernel<704>")
        assert_not_ran(names, "agg_mid_kernel")


# ------------------------------------------------------------------ FASTREG
@pytest.mark.parametrize("form", ["kw1_1", "kw1_2", "kw1_4", "kw4", "kw0s", "kw0u"])
@pytest.mark.parametrize("slots", [4, 8])
@pytest.mark.parametrize("nsum", [1, 2, 3, 4, 5, 6])
def test_fastreg_kernels(ctx, nsum, slots, form):
    """the register path for every NSUM, both slot counts and the three key decoders.  4 groups run the 4-slot kernel
    on the whole input; 7 groups run it on the probe chunk (3 groups miss its slots and take the global path) and the
    8-slot kernel on the rest.  INT64 / UINT64 inputs carry every edge value on both sides of the 2^40 limit."""
    rng = np.random.default_rng(nsum * 100 + slots * 10 + len(form))
    ng = 4 if slots == 4 else 7
    n = PROBE + 70_001
    gid = rng.integers(0, ng, size=n)
    keys = key_columns(form, gid, ng)
    inputs = sum_inputs(rng, nsum, n)
    names = agg_run(ctx, keys, gid, ng, inputs, sum_aggs(nsum))
    for s in (4, 8) if slots == 8 else (4,):
        assert_ran(names, f"agg_fastreg_kernel<{nsum}, {s}, {fastreg_threads(s, nsum)}, {fastreg_kw(form)}>")
    assert_not_ran(names, "agg_fast_kernel", "agg_mid_kernel", "agg_priv_kernel", "agg_wpriv_kernel")


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, PROBE - 1, PROBE + 1, 6_000_001])
def test_fastreg_row_counts(ctx, n):
    """row counts around the 1024-row tile, the 256 K-row probe chunk (one row after it) and one batch of 6 M rows
    (every CTA walks many tiles; UINT64 2^64 - 1 and INT64 extremes in every group)"""
    rng = np.random.default_rng(n)
    ng = min(n, 3) if n <= PROBE else 6
    gid = rng.integers(0, ng, size=n)
    keys = key_columns("kw1_2", gid, ng)
    inputs = sum_inputs(rng, 3, n)
    names = agg_run(ctx, keys, gid, ng, inputs, sum_aggs(3))
    assert_ran(names, "agg_fastreg_kernel<3, 4, 224, 1>")
    if n > PROBE:
        assert_ran(names, "agg_fastreg_kernel<3, 8, 192, 1>")
    assert_not_ran(names, "agg_fast_kernel", "agg_mid_kernel")


# ------------------------------------------------------------------ FAST
def small_keys(rng, gid, null_keys):
    """UTINYINT x SMALLINT keys; with null_keys the last group's first key is NULL"""
    k1 = (gid % 4).astype(np.uint8)
    k2 = (gid // 4 * 1000 - 3000).astype(np.int16)
    kv = (gid != gid.max()) if null_keys else None
    return [(k1, kv), (k2, None)]


@pytest.mark.parametrize("ng", [6, 13, 20])
@pytest.mark.parametrize("shape", ["null_keys", "nullable_inputs", "minmax", "narrow_inputs", "float_sums"])
def test_fast_kernel_shapes(ctx, shape, ng):
    """shapes the register path refuses run the shared-memory FAST kernel: NULL keys, nullable inputs, MIN / MAX, 1- to
    4-byte inputs, FLOAT / DOUBLE sums.  13 and 20 groups overflow a directory of 8 or 16 slots (the rest go to the
    global path inline).  Probe-sized inputs, so that FAST is the only shared-memory kernel."""
    rng = np.random.default_rng(len(shape) * 100 + ng)
    n = 150_000
    gid = rng.integers(0, ng, size=n)
    keys = small_keys(rng, gid, shape == "null_keys")
    a = planted(rng, np.int64, n, -2 ** 39, 2 ** 39)
    b = planted(rng, np.uint64, n, 0, 2 ** 40)
    inputs = [(a, None), (b, None)]
    aggs = [("sum", 0), ("avg", 0), ("sum", 1), ("count", 1), ("count_star", -1)]
    if shape == "nullable_inputs":
        inputs = [(a, rng.random(n) > 0.3), (b, rng.random(n) > 0.5)]
    elif shape == "minmax":
        aggs += [("min", 0), ("max", 0), ("min", 1), ("max", 1)]
    elif shape == "narrow_inputs":
        inputs = [(rng.integers(-128, 128, size=n).astype(np.int8), None),
                  (rng.integers(0, 2 ** 16, size=n).astype(np.uint16), None),
                  (rng.integers(-2 ** 31, 2 ** 31, size=n).astype(np.int32), None),
                  (rng.integers(0, 2 ** 32, size=n).astype(np.uint32), None)]
        aggs = [("sum", 0), ("avg", 0), ("sum", 1), ("sum_no_overflow", 2), ("sum", 3), ("avg", 3), ("count_star", -1)]
    elif shape == "float_sums":
        inputs = [(rng.standard_normal(n) * 1e6, None), (rng.standard_normal(n).astype(np.float32), None), (a, None)]
        aggs = [("sum", 0), ("avg", 0), ("sum", 1), ("sum", 2), ("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_ran(names, "agg_fast_kernel")
    assert_not_ran(names, "agg_fastreg_kernel", "agg_mid_kernel", "agg_priv_kernel", "agg_wpriv_kernel")


def test_fast_partial_overflow(ctx):
    """per-thread 64-bit partials of FAST that wrap: INT64 values near 2^62 (a partial overflows every other row) and
    UINT64 2^64 - 1 repeated; the partial is pushed to the global state before it wraps (the `ovf` branch)"""
    rng = np.random.default_rng(5)
    n, ng = 200_000, 5
    gid = rng.integers(0, ng, size=n)
    keys = small_keys(rng, gid, True)
    a = rng.integers(2 ** 62 - 1000, 2 ** 62 + 1, size=n, dtype=np.int64)
    a[gid == 1] = -a[gid == 1]
    b = np.full(n, 2 ** 64 - 1, dtype=np.uint64)
    b[rng.integers(0, n, size=1000)] = np.uint64(2 ** 63)
    inputs = [(a, None), (b, None)]
    aggs = [("sum", 0), ("avg", 0), ("sum_no_overflow", 0), ("sum", 1), ("avg", 1), ("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_ran(names, "agg_fast_kernel")
    assert_not_ran(names, "agg_fastreg_kernel", "agg_mid_kernel")


INT_TYPES = [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64]
DOUBLE_SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e308, -1e308, 5e-324])


@pytest.mark.parametrize("half", [0, 1])
@pytest.mark.parametrize("path", ["fast", "mid"])
def test_minmax_type_limits(ctx, path, half):
    """MIN / MAX / SUM over every integer width at its limits (four widths per case: an aggregate holds at most 16
    aggregates), and MIN / MAX over doubles with +-0.0, +-inf and NaN (NaN orders above everything; a group whose only
    values are NaN) and over FLOAT, against oracle.port.group_by, on FAST (5 groups) and on MID (an 8-byte key: the
    shared-memory table from the first row)"""
    rng = np.random.default_rng(11 + 2 * half if path == "fast" else 12 + 2 * half)
    n, ng = 30_000, 5
    gid = rng.integers(0, ng, size=n)
    if path == "fast":
        keys = [((gid * 3 - 6).astype(np.int8), None)]
    else:
        keys = [(gid.astype(np.int64) * -(2 ** 50) + 1, None)]
    inputs, aggs = [], []
    for dt in INT_TYPES[4 * half: 4 * half + 4]:
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, size=n, endpoint=True, dtype=dt)
        v[rng.integers(0, n, size=30)] = info.min
        v[rng.integers(0, n, size=30)] = info.max
        valid = rng.random(n) > 0.1 if dt in (np.int16, np.uint64) else None
        i = len(inputs)
        inputs.append((v, valid))
        aggs += [("min", i), ("max", i), ("sum", i)]
    d = rng.standard_normal(n) * 1e3
    pick = rng.random(n) < 0.05
    d[pick] = rng.choice(DOUBLE_SPECIALS, size=int(pick.sum()))
    d[gid == 3] = np.nan                                          # a group of NaNs only
    if half == 0:
        inputs.append((d, None))
    else:
        inputs.append((rng.choice(np.array([0.0, -0.0, 1.5, -2.5, np.inf], dtype=np.float32), size=n),
                       rng.random(n) > 0.2))
    aggs += [("min", len(inputs) - 1), ("max", len(inputs) - 1), ("count", len(inputs) - 1)]
    exp_keys = [(k, kv) for k, kv in keys]
    oracle_aggs = [(fn, inputs[i] if i >= 0 else None) for fn, i in aggs]
    oracle = P.group_by(exp_keys, oracle_aggs, n)
    exp = {tuple(canon(x) if x is not None else None for x in k): v for k, v in oracle.items()}
    names = agg_run(ctx, keys, gid, ng, inputs, aggs, exp=exp)
    if path == "fast":
        assert_ran(names, "agg_fast_kernel")
        assert_not_ran(names, "agg_mid_kernel", "agg_fastreg_kernel")
    else:
        assert_ran(names, "agg_mid_kernel")
        assert_not_ran(names, "agg_fast_kernel", "agg_fastreg_kernel", "agg_priv_kernel")


# ------------------------------------------------------------------ PRIV / WPRIV
PRIV_KNOBS = {"wpriv": {"B200_AGG_WPRIV": "1"}, "priv": {"B200_AGG_NO_WPRIV": "1"},
              "directory": {"B200_AGG_NO_DIRECT": "1"}, "priv2": {"B200_AGG_PRIV": "2", "B200_AGG_NO_WPRIV": "1"}}


def set_knobs(monkeypatch, knob):
    for k, v in PRIV_KNOBS[knob].items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("knob,ng,nsum,form", [
    ("wpriv", 35, 1, "kw1_2"), ("wpriv", 35, 6, "kw1_2"), ("wpriv", 600, 2, "kw1_2"), ("wpriv", 40, 3, "kw0s"),
    ("priv", 35, 1, "kw1_2"), ("priv", 9, 5, "kw1_2"), ("priv", 35, 3, "kw0u"),
    ("directory", 35, 2, "kw1_2"), ("directory", 20, 1, "kw4"), ("directory", 24, 4, "kw0s"),
    ("priv2", 6, 2, "kw1_2"), ("priv", 600, 1, "kw1_2")])
def test_priv_kernels(ctx, monkeypatch, knob, ng, nsum, form):
    """the private-accumulator paths after the adaptation probe: warp-private (B200_AGG_WPRIV=1) and thread-private
    (B200_AGG_NO_WPRIV) copies on the direct slot tables built from the probe's groups (agg_list_keys_kernel), the
    directory lookup (B200_AGG_NO_DIRECT: one-byte, 4-byte and generic key decoders), and PRIV for <= 8 groups
    (B200_AGG_PRIV=2).  Thread-private copies of 600 slots do not fit shared memory: without WPRIV that shape falls
    back to MID."""
    set_knobs(monkeypatch, knob)
    rng = np.random.default_rng(ng * 10 + nsum + len(form))
    n = PROBE + 400_003
    gid = rng.integers(0, ng, size=n)
    keys = key_columns(form, gid, ng)
    inputs = sum_inputs(rng, nsum, n)
    names = agg_run(ctx, keys, gid, ng, inputs, sum_aggs(nsum))
    if knob == "priv" and ng == 600:
        assert_ran(names, "agg_list_keys_kernel", "agg_mid_kernel")
        assert_not_ran(names, "agg_priv_kernel", "agg_wpriv_kernel")
        return
    assert_not_ran(names, "agg_mid_kernel", "agg_fast_kernel")
    if knob == "wpriv":
        assert_ran(names, f"agg_wpriv_kernel<{nsum}>", "agg_list_keys_kernel")
        assert_not_ran(names, "agg_priv_kernel")
    elif knob in ("priv", "priv2"):
        assert_ran(names, f"agg_priv_kernel<{nsum}, 2>", "agg_list_keys_kernel")
        assert_not_ran(names, "agg_wpriv_kernel")
    else:
        assert_ran(names, f"agg_priv_kernel<{nsum}, {fastreg_kw(form)}>")
        assert_not_ran(names, "agg_wpriv_kernel", f"agg_priv_kernel<{nsum}, 2>")


@pytest.mark.parametrize("knob", ["wpriv", "priv", "directory"])
@pytest.mark.parametrize("case", ["tinyint_span_zero", "integer_span_zero", "late_keys", "four_keys"])
def test_priv_direct_edges(ctx, monkeypatch, knob, case):
    """direct slot addressing at its edges.  Signed keys spanning zero: the code tables are built from the raw bit
    patterns, so TINYINT {-3..3} spans the byte range 0..255 (direct), INTEGER {-3..3} spans 2^32 values (no direct
    tables: the directory kernel takes it whatever the knob).  Keys first seen after the 256 K-row probe: inside a
    code table's range but absent from it, outside the range, and (directory) beyond the slot slack - all must reach
    the global path and still be counted.  Four key columns (the most direct addressing takes)."""
    set_knobs(monkeypatch, knob)
    rng = np.random.default_rng(len(case) * 7 + len(knob))
    n = PROBE + 500_000
    if case in ("tinyint_span_zero", "integer_span_zero"):
        ng = 35
        gid = rng.integers(0, ng, size=n)
        dt = np.int8 if case == "tinyint_span_zero" else np.int32
        keys = [((gid % 7 - 3).astype(dt), None), ((gid // 7).astype(np.uint8), None)]
        kw = 1 if dt == np.int8 else 0
    elif case == "four_keys":
        ng = 36
        gid = rng.integers(0, ng, size=n)
        keys = [((gid % 2).astype(np.uint8), None), ((gid // 2 % 3 - 1).astype(np.int8), None),
                ((gid // 6 % 2 * 200).astype(np.uint8), None), ((gid // 12 - 1).astype(np.int8), None)]
        kw = 1
    else:
        # the probe sees 20 groups, keys 0, 2, .., 38; later rows add 1, 3, .., 37 (inside the code table's range but
        # absent from it), 39 and 200 .. 219 (outside it): 40 new keys, far more than the directory's slot slack
        ng = 60
        gid = rng.integers(0, 20, size=n)
        late = np.arange(PROBE, n)
        gid[late] = rng.integers(0, ng, size=len(late))
        k = np.where(gid < 20, gid * 2, np.where(gid < 40, (gid - 20) * 2 + 1, 160 + gid)).astype(np.uint8)
        keys = [(k, None)]
        kw = 1
    inputs = sum_inputs(rng, 2, n)
    names = agg_run(ctx, keys, gid, ng, inputs, sum_aggs(2))
    assert_not_ran(names, "agg_mid_kernel", "agg_fast_kernel")
    direct = case != "integer_span_zero" and knob != "directory"
    if not direct:
        assert_ran(names, f"agg_priv_kernel<2, {kw}>")
        assert_not_ran(names, "agg_wpriv_kernel", "agg_priv_kernel<2, 2>")
    elif knob == "wpriv":
        assert_ran(names, "agg_wpriv_kernel<2>")
        assert_not_ran(names, "agg_priv_kernel")
    else:
        assert_ran(names, "agg_priv_kernel<2, 2>")
        assert_not_ran(names, "agg_wpriv_kernel")


# ------------------------------------------------------------------ MID / MID2
@pytest.mark.parametrize("shape", ["nullable_1word", "int64_key", "int64_int32_key"])
def test_mid_kernel(ctx, shape):
    """the shared-memory hash table: a 1-word key (INTEGER) with nullable inputs and 300 groups (after the probe; the
    private paths take neither NULLs nor MIN / MAX), and 2-word keys (INT64 + the NULL-flag byte, INT64 + INTEGER) that
    take MID from the first row; MIN / MAX / SUM over doubles and several integer widths, COUNT of nullable inputs"""
    rng = np.random.default_rng(len(shape))
    n = PROBE + 300_001
    ng = 300 if shape == "nullable_1word" else 50
    gid = rng.integers(0, ng, size=n)
    if shape == "nullable_1word":
        keys = [((gid * 11 - 1500).astype(np.int32), None)]
    elif shape == "int64_key":
        keys = [(gid.astype(np.int64) * 2 ** 45 - 2 ** 62, None)]
    else:
        keys = [(gid.astype(np.int64) * -(2 ** 33), None), ((gid % 3 - 1).astype(np.int32), None)]
    a = planted(rng, np.int64, n, -2 ** 62, 2 ** 62)
    b = planted(rng, np.uint64, n, 0, 2 ** 64 - 1)
    c = rng.integers(-2 ** 31, 2 ** 31, size=n).astype(np.int32)
    h = rng.integers(0, 2 ** 16, size=n).astype(np.uint16)
    inputs = [(a, rng.random(n) > 0.3), (b, None), (c, rng.random(n) > 0.1), (h, None)]
    aggs = [("sum", 0), ("avg", 0), ("count", 0), ("min", 0), ("max", 0), ("sum", 1), ("max", 1), ("min", 1),
            ("sum", 2), ("min", 2), ("count", 2), ("sum", 3), ("max", 3), ("count_star", -1)]
    if shape != "nullable_1word":
        inputs.append((rng.standard_normal(n) * 1e3, None))
        aggs += [("sum", 4), ("avg", 4)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_ran(names, "agg_mid_kernel")
    assert_not_ran(names, "agg_priv_kernel", "agg_wpriv_kernel", "agg_fastreg_kernel", "agg_mid2_kernel")


@pytest.mark.parametrize("ninputs", [9, 10])
def test_more_columns_than_a_tile_stage_takes(ctx, ninputs):
    """DuckDB hands every aggregate its own copy of the input column, so ten aggregates over nullable inputs with a
    nullable key stage 22 columns, two more than a tile stage holds (TP_MAX_COLS).  Such a batch must go to the
    generic sink kernel: it used to be dispatched to the MID path, which refused it ("too many staged columns") and
    failed the query.  Nine inputs (20 columns) still fit and take MID."""
    rng = np.random.default_rng(ninputs)
    n, ng = PROBE + 50_001, 35
    gid = rng.integers(0, ng, size=n)
    keys = [((gid * 7 - 100).astype(np.int32), gid != 0)]   # group 0 is the NULL key
    inputs = [(rng.integers(-2 ** 31, 2 ** 31, size=n).astype(np.int32), rng.random(n) > 0.2) for _ in range(ninputs)]
    aggs = [("sum", i) for i in range(ninputs)] + [("count", 0), ("min", 1), ("max", 2), ("avg", 3), ("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    if ninputs == 10:
        assert_ran(names, "agg_sink_kernel")
        assert_not_ran(names, "agg_mid_kernel", "agg_mid2_kernel", "agg_priv_kernel", "agg_wpriv_kernel",
                       "agg_fastreg_kernel")
    else:
        assert_ran(names, "agg_mid_kernel")


def test_mid_spill(ctx):
    """more groups than the shared table's fill limit: five inputs with SUM, MIN and MAX make a slot 188 bytes, the
    table shrinks to 512 slots (384 usable), and of 650 groups the rows of the others spill to the global path"""
    rng = np.random.default_rng(21)
    n, ng = PROBE + 100_000, 650
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.int64) * 3 - 900, None)]
    inputs, aggs = [], []
    for dt in [np.int8, np.uint16, np.int32, np.uint64, np.int64]:
        info = np.iinfo(dt)
        inputs.append((rng.integers(info.min, info.max, size=n, endpoint=True, dtype=dt), None))
        aggs += [("sum", len(inputs) - 1), ("min", len(inputs) - 1), ("max", len(inputs) - 1)]
    aggs += [("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_ran(names, "agg_mid_kernel")


@pytest.mark.parametrize("minmax", [False, True])
def test_mid_not_for_long_keys(ctx, minmax):
    """a key of more than 2 words (INT64 x 2 + TINYINT: 3 words) does not fit the shared table: the high-cardinality
    table takes it, or with MIN / MAX (which that table does not hold) the global row kernel"""
    rng = np.random.default_rng(31 + minmax)
    n, ng = 300_000, 40
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.int64) * 2 ** 40, None), (-gid.astype(np.int64), None), ((gid % 5).astype(np.int8), None)]
    inputs = [(planted(rng, np.int64, n, -2 ** 50, 2 ** 50), None)]
    aggs = [("sum", 0), ("avg", 0), ("count_star", -1)] + ([("min", 0), ("max", 0)] if minmax else [])
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_not_ran(names, *NOT_LOW_CARD)
    if minmax:
        assert_ran(names, "agg_sink_kernel")
    else:
        assert_ran(names, "agg_hc_direct_kernel<3, 1>")


@pytest.mark.parametrize("nc", [512, 704, 960])
def test_mid2_kernel(ctx, monkeypatch, nc):
    """the carry-free limb variant (B200_AGG_MID2=<threads>): values at +-(2^40 - 1) inside the limbs' range, and -2^40
    - 1, 2^40, the INT64 extremes just outside (global path, the row applied there entirely); UINT64 at and beyond
    2^40; a nullable INTEGER input (its count kept per slot)"""
    monkeypatch.setenv("B200_AGG_MID2", str(nc))
    rng = np.random.default_rng(nc)
    n, ng = 1_000_003, 6
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.int64) - 3, None)]
    a = rng.choice(np.array([2 ** 40 - 1, -(2 ** 40 - 1), 2 ** 40 - 2, 0, -1], dtype=np.int64), size=n)
    for e in SIGNED_EDGES:
        a[rng.integers(0, n, size=50)] = e
    b = planted(rng, np.uint64, n, 0, 2 ** 40)
    c = rng.integers(-2 ** 31, 2 ** 31, size=n).astype(np.int32)
    inputs = [(a, None), (b, None), (c, rng.random(n) > 0.25)]
    aggs = [("sum", 0), ("avg", 0), ("sum", 1), ("sum", 2), ("count", 2), ("avg", 2), ("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs)
    assert_ran(names, f"agg_mid2_kernel<{nc}>")
    assert_not_ran(names, "agg_mid_kernel")


def test_mid2_periodic_flushes(ctx, monkeypatch):
    """40 M rows: every CTA of MID2 crosses its periodic flush (every 2^18 rows of the CTA: a limb word absorbs 2^18
    additions before it could wrap) as well as the final one; one group gets only values at 2^40 - 1 (every limb at
    its maximum).  A UTINYINT key with a nullable input: FAST on the probe, then MID (PRIV refuses NULLs)."""
    monkeypatch.setenv("B200_AGG_MID2", "704")
    rng = np.random.default_rng(40)
    n, ng = 40_000_000, 12
    gid = rng.integers(0, ng, size=n).astype(np.uint8)
    keys = [(gid, None)]
    a = rng.integers(-2 ** 40 + 1, 2 ** 40, size=n, dtype=np.int64)
    a[gid == 0] = 2 ** 40 - 1
    a[gid == 1] = -(2 ** 40 - 1)
    valid = np.ones(n, dtype=bool)
    valid[rng.integers(0, n, size=n // 10)] = False
    inputs = [(a, valid)]
    aggs = [("sum", 0), ("count", 0), ("count_star", -1)]
    names = agg_run(ctx, keys, gid.astype(np.int64), ng, inputs, aggs)
    assert_ran(names, "agg_mid2_kernel<704>")
    assert_not_ran(names, "agg_mid_kernel")


# ------------------------------------------------------------------ generic table (agg.cu)
def test_generic_table_growth_and_replay(ctx):
    """a 4-group probe chunk fixes the 4-slot register path; then 200 K new groups arrive: their rows miss the slots,
    go to the generic table, find it at its fill limit, are deferred; the table grows (rehash) and they are replayed
    by the row kernel.  Finalize reads the generic table."""
    rng = np.random.default_rng(3)
    n, ng = PROBE + 1_000_000, 200_004
    gid = np.concatenate([rng.integers(0, 4, size=PROBE), rng.integers(0, ng, size=n - PROBE)])
    keys = [((gid * 13 - 1_000_000).astype(np.int32), None)]
    inputs = sum_inputs(rng, 2, n)
    names = agg_run(ctx, keys, gid, ng, inputs, sum_aggs(2))
    assert_ran(names, "agg_fastreg_kernel<2, 4, 224, 4>", "agg_sink_kernel", "agg_rehash_kernel", "agg_init_kernel",
               "agg_finalize_kernel", "fill_u64_kernel3")


@pytest.mark.parametrize("path", ["fastreg", "priv", "mid", "hc"])
def test_validity_arrives_later(ctx, monkeypatch, path):
    """an input that arrives WITHOUT a validity mask in batch 1 and with one from batch 2 (x) or batch 3 (y) on: cnt(x)
    starts being tracked then and is brought up to the row count (agg_fix_cnt_kernel), so COUNT(x) and the NULL-ness of
    SUM(x) still count batch 1's rows.  Group 0's later rows are all NULL (SUM stays non-NULL); one group only shows
    up after batch 1 with nothing but NULLs (SUM is NULL, COUNT 0)."""
    rng = np.random.default_rng(len(path))
    if path == "fastreg":
        ng, n = 4, 600_000
        keys_of = lambda g: [((g % 2).astype(np.uint8), None), ((g // 2).astype(np.uint8), None)]  # noqa: E731
    elif path == "priv":
        monkeypatch.setenv("B200_AGG_WPRIV", "1")
        ng, n = 35, 1_200_000
        keys_of = lambda g: [((g % 7).astype(np.uint8), None), ((g // 7).astype(np.uint8), None)]  # noqa: E731
    elif path == "mid":
        ng, n = 50, 600_000
        keys_of = lambda g: [(g.astype(np.int64) * 2 ** 50, None)]  # noqa: E731
    else:
        ng, n = 100_000, 1_600_000
        keys_of = lambda g: [((g * 7 - 10 ** 6).astype(np.int32), None)]  # noqa: E731
    bounds = [0, n // 2, 3 * n // 4, n]
    gid = rng.integers(1, ng - 1, size=n)
    gid[rng.integers(0, n, size=200)] = 0
    gid[rng.integers(bounds[1], n, size=100)] = ng - 1            # the late group: rows only after batch 1
    keys = keys_of(gid)
    x = planted(rng, np.int64, n, -2 ** 39, 2 ** 39)
    y = planted(rng, np.uint64, n, 0, 2 ** 40)
    xv = np.ones(n, dtype=bool)
    xv[bounds[1]:] = rng.random(n - bounds[1]) > 0.3
    yv = np.ones(n, dtype=bool)
    yv[bounds[2]:] = rng.random(n - bounds[2]) > 0.5
    for v in (xv, yv):
        v[(gid == 0) & (np.arange(n) >= bounds[1])] = False
        v[gid == ng - 1] = False
    yv[:bounds[2]] = True
    inputs = [(x, xv), (y, yv)]
    masked = [[False, False], [True, False], [True, True]]
    aggs = [("sum", 0), ("count", 0), ("avg", 0), ("sum", 1), ("count", 1), ("count_star", -1)]
    names = agg_run(ctx, keys, gid, ng, inputs, aggs, bounds=bounds, masked=masked)
    assert_ran(names, "agg_fix_cnt_kernel", {"fastreg": "agg_fastreg_kernel<2, 4, 224, 1>", "priv": "agg_wpriv_kernel<2>",
                                             "mid": "agg_mid_kernel", "hc": "agg_hc_direct_kernel<1, 2>"}[path])


def exported_parts(ctx, keys, inputs, aggs, parts):
    """one aggregate per row range, sunk and left open"""
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]
    out = []
    for lo, hi in parts:
        a = ops.HashAggregate(ctx, key_types, descs_of(aggs, inputs))
        if hi > lo:
            sink_all(ctx, a, [(k[lo:hi], None if kv is None else kv[lo:hi]) for k, kv in keys],
                     [(v[lo:hi], None if m is None else m[lo:hi]) for v, m in inputs], [0, hi - lo])
        out.append(a)
    return out


@pytest.mark.parametrize("path", ["fastreg", "priv", "mid"])
def test_export_combine_states(ctx, monkeypatch, path):
    """partial aggregates whose groups live in a FASTREG, PRIV or MID table, exported as state columns and combined
    into one aggregate: equal to one aggregate over all rows"""
    monkeypatch.setenv("B200_AGG_WPRIV", "1")
    rng = np.random.default_rng(60 + len(path))
    ng, n = {"fastreg": (4, 300_000), "priv": (35, 1_000_000), "mid": (40, 400_000)}[path]
    gid = rng.integers(0, ng, size=n)
    keys = (key_columns("kw1_2", gid, ng) if path != "mid" else [(gid.astype(np.int64) * 2 ** 41 - 7, None)])
    inputs = sum_inputs(rng, 2, n)
    aggs = sum_aggs(2)
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]

    def run():
        parts = exported_parts(ctx, keys, inputs, aggs, [(0, n // 2), (n // 2, n)])
        final = ops.HashAggregate(ctx, key_types, descs_of(aggs, inputs))
        for a in parts:
            final.combine_states(a.export_states())
            a.close()
        out = fetch_groups(final.finalize(), len(keys), len(aggs))
        final.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel"])
    assert_same(got, reference(keys, gid, ng, inputs, aggs), aggs, inputs)
    assert_ran(names, "agg_export_kernel", "agg_combine_kernel",
               {"fastreg": "agg_fastreg_kernel<2, 4, 224, 1>", "priv": "agg_wpriv_kernel<2>", "mid": "agg_mid_kernel"}[path])


def packed_case(rng, n):
    """DOUBLE keys with -0.0 / 0.0 and NaNs of two payloads (one group each), a nullable INTEGER key; integer and
    double inputs"""
    vals = np.array([0.0, -0.0, np.nan, -np.nan, 1.5, -7.25, np.inf])
    k1 = rng.choice(vals, size=n)
    k2 = rng.integers(-2, 3, size=n).astype(np.int32)
    k2v = rng.random(n) > 0.1
    x = rng.integers(-2 ** 50, 2 ** 50, size=n, dtype=np.int64)  # (sums below 2^63: the oracle's AVG is exact)
    d = rng.standard_normal(n)
    inputs = [(x, rng.random(n) > 0.2), (d, None)]
    aggs = [("sum", 0), ("avg", 0), ("count", 0), ("min", 0), ("max", 1), ("sum", 1), ("count_star", -1)]
    return [(k1, None), (k2, k2v)], inputs, aggs


def test_packed_three_ranks(ctx):
    """three partial aggregates packed into consecutive slices of one device buffer (what an all-gather leaves) and
    combined: an empty rank, ranks with a NULL-key group, DOUBLE keys with -0.0 / NaN.  Equal to one aggregate over all
    rows (oracle.port.group_by)."""
    import torch

    rng = np.random.default_rng(70)
    n = 40_000
    keys, inputs, aggs = packed_case(rng, n)
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]
    max_groups = 64

    def run():
        parts = exported_parts(ctx, keys, inputs, aggs, [(0, n // 3), (n // 3, n // 3), (n // 3, n)])
        words = parts[0].packed_words(max_groups)
        buf = torch.zeros(3 * words, dtype=torch.int64, device="cuda:0")
        for r, a in enumerate(parts):
            a.export_packed(buf.data_ptr() + r * words * 8, max_groups)
        final = ops.HashAggregate(ctx, key_types, descs_of(aggs, inputs))
        final.combine_packed(buf.data_ptr(), 3, max_groups)
        ctx.sync()
        out = fetch_groups(final.finalize(), len(keys), len(aggs))
        for a in parts + [final]:
            a.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel"])
    oracle = P.group_by(keys, [(f, inputs[i] if i >= 0 else None) for f, i in aggs], n)
    exp = {tuple(canon(x) if x is not None else None for x in k): v for k, v in oracle.items()}
    assert any(k[1] is None for k in exp), "the data must hold a NULL-key group"
    assert_same(got, exp, aggs, inputs)
    assert_ran(names, "agg_export_packed_kernel", "agg_packed_header_kernel", "agg_combine_packed_kernel")


def test_packed_overflow_is_reported(ctx):
    """a rank with more groups than max_groups sets its overflow flag; combining it makes finalize fail with
    ERR_CAPACITY instead of returning a partial answer"""
    import torch

    rng = np.random.default_rng(71)
    n = 10_000
    keys, inputs, aggs = packed_case(rng, n)
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]
    max_groups = 8  # each half holds 5 x 6 groups

    def run():
        parts = exported_parts(ctx, keys, inputs, aggs, [(0, n // 2), (n // 2, n)])
        words = parts[0].packed_words(max_groups)
        buf = torch.zeros(2 * words, dtype=torch.int64, device="cuda:0")
        final = ops.HashAggregate(ctx, key_types, descs_of(aggs, inputs))
        for r, a in enumerate(parts):
            a.export_packed(buf.data_ptr() + r * words * 8, max_groups)
        final.combine_packed(buf.data_ptr(), 2, max_groups)
        ctx.sync()
        flags = buf.view(2, words)[:, :2].cpu().numpy()
        with pytest.raises(capi.B200Error) as e:
            final.finalize()
        for a in parts + [final]:
            a.close()
        return flags, e.value.code

    (flags, code), names = traced_window(run, always=["agg_init_kernel"])
    assert (flags[:, 0] == max_groups).all() and (flags[:, 1] == 1).all(), flags
    assert code == capi.ERR_CAPACITY
    assert_ran(names, "agg_combine_packed_kernel")
