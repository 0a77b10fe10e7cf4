"""Every fast-path kernel variant of the filter, high-cardinality aggregate and lean join probe, forced by its shape or
knob, checked against the oracle AND against the kernel trace: each dispatcher falls back silently to a generic kernel
when a variant is not eligible, and the fall-back computes the same answer, so without the trace a test written for a
fast kernel could be testing the interpreter.  Integer results bit-exact; AVG within 1e-15 relative."""
import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran, kernel_trace, ran, traced
from oracle import port as P
from test_gpu_parity import build_expr, run_filter, run_join

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of filter_tile.cu, agg_hc.cu, join_tile.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "filter_mask_tile_kernel": ["test_filter_single_term_limits", "test_filter_and_trees"],
    "compact_tile_kernel": ["test_filter_single_term_limits", "test_filter_projection_widths"],
    "filter_fused_tile_kernel": ["test_filter_and_trees", "test_filter_projection_widths"],
    "agg_hc_direct_kernel": ["test_hc_kernels"],
    "agg_hc_simple_kernel": ["test_hc_kernels"],
    "agg_hc_kernel": ["test_hc_kernels", "test_hc_nullable"],
    "agg_hc_rows_kernel": ["test_hc_growth_batches", "test_hc_dictionary_keys"],
    "agg_hc_flush_kernel": ["test_hc_export_combine"],
    "agg_hc_absorb_kernel": ["test_hc_kernels"],
    "agg_hc_finalize_kernel": ["test_hc_kernels"],
    "agg_hc_rehash_kernel": ["test_hc_growth_batches"],
    "hc_count_kernel": ["test_hc_kernels"],
    "hc_spread_count_kernel": ["test_hc_growth_batches"],
    "join_probe_lean2_kernel": ["test_join_lean_probe"],
    "join_probe_tile_kernel": ["test_join_lean1_and_control"],
}
# kernels of those files that no test here has to reach, with the reason
KERNEL_EXCLUDED = {}

INT_DTYPES = [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64]
CMP_OPS = ["eq", "ne", "lt", "gt", "le", "ge"]


def test_kernel_trace_sees_library_kernels(ctx):
    """the trace must see kernels libduckdb_b200.so launches through ctypes; every other assertion here relies on it"""
    b = ops.Batch.upload(ctx, [ops.Vector.flat(np.arange(1000, dtype=np.int64))], 1000)
    import torch
    out = torch.empty(1000, dtype=torch.int64, device="cuda:0")
    with kernel_trace() as names:
        ops.hash_keys(ctx, b, [0], out.data_ptr())
        ctx.sync()
    assert names, "torch.profiler recorded no CUDA kernel at all: CUPTI activity tracing is not available here"
    assert ran(names, "hash_kernel"), f"the trace misses the library's hash_kernel; it holds {sorted(set(names))}"


# ------------------------------------------------------------------ filter
def mask_tile_kernel(widths):
    """filter_mask_tile_kernel<MROWS>: the largest super-tile (32, 16 or 8 rows per thread) whose three stages of the
    predicate's distinct columns fit 50 KB"""
    w = sum(widths)
    return f"filter_mask_tile_kernel<{32 if w <= 2 else 16 if w <= 4 else 8}>"


def check_filter(ctx, cols, n, pred, projs=(), bitmap=False):
    """run the program, compare selection, mask and projected columns with the oracle; -> surviving row count"""
    exp_sel, keep = P.filter_select(pred, cols, n)
    vectors = [ops.Vector.flat(v, np.ones(n, dtype=bool) if bitmap else None) for v, _ in cols]
    count, sel, mask, outs = run_filter(ctx, None, n, pred, projs, vectors=vectors)
    assert count == len(exp_sel), (pred, n, count, len(exp_sel))
    np.testing.assert_array_equal(sel, exp_sel)
    np.testing.assert_array_equal(capi.valid_from_words(mask, n), keep)
    if n % 64:
        assert int(mask[-1]) >> (n % 64) == 0
    for (v, valid), p in zip(outs, projs):
        np.testing.assert_array_equal(v, cols[p[1]][0][exp_sel])
        assert valid.all()
    return count


def edge_column(rng, dtype, n):
    info = np.iinfo(dtype)
    v = rng.integers(info.min, info.max, size=n, endpoint=True, dtype=dtype)
    edges = np.array([info.min, info.min + 1, info.max - 1, info.max, 0], dtype=dtype)
    v[rng.integers(0, n, size=200)] = rng.choice(edges, size=200)
    return v


@pytest.mark.parametrize("dtype", INT_DTYPES)
def test_filter_single_term_limits(ctx, monkeypatch, dtype):
    """`col CMP const` and `const CMP col` for all six operators with constants at MIN, MIN+1, MAX-1, MAX, 0 and a
    value from the data, in every integer width and signedness: the TMA mask kernel (range form on full tiles, the
    single-term super-tile loop, the per-row form on the ragged tail) with the TMA compaction, the fused single-pass
    kernel, and the interpreter (the same columns with an all-valid bitmap) must all equal the oracle.  Constants just
    outside the type are rejected by both paths."""
    rng = np.random.default_rng(np.dtype(dtype).itemsize * 2 + (np.dtype(dtype).kind == "u"))
    info = np.iinfo(dtype)
    n = 40123  # full super-tiles of every width plus a ragged one
    v = edge_column(rng, dtype, n)
    cols = [(v, None)]
    consts = [int(info.min), int(info.min) + 1, int(info.max) - 1, int(info.max), 0, int(v[17])]
    preds = []
    for op in CMP_OPS:
        for c in consts:
            preds.append((op, ("col", 0), ("const", c, dtype)))
            preds.append((op, ("const", c, dtype), ("col", 0)))
    width = np.dtype(dtype).itemsize
    for mode in ("tile", "fused", "bitmap"):
        if mode == "fused":
            monkeypatch.setenv("B200_FILTER_FUSED", "1")
        else:
            monkeypatch.delenv("B200_FILTER_FUSED", raising=False)
        with kernel_trace() as names:
            for pred in preds:
                check_filter(ctx, cols, n, pred, [("col", 0)], bitmap=mode == "bitmap")
        if mode == "tile":
            assert_ran(names, mask_tile_kernel([width]), "compact_tile_kernel")
            assert_not_ran(names, "filter_mask_kernel", "compact_kernel", "filter_fused_tile_kernel")
        elif mode == "fused":
            assert_ran(names, "filter_fused_tile_kernel")
            assert_not_ran(names, "filter_mask_kernel", "filter_mask_tile_kernel", "compact_tile_kernel")
        else:
            assert_ran(names, "filter_mask_kernel", "compact_kernel<false>")
            assert_not_ran(names, "filter_mask_tile_kernel", "compact_tile_kernel", "filter_fused_tile_kernel")
        if width < 8:
            for c in (int(info.min) - 1, int(info.max) + 1):
                for pred in (("lt", ("col", 0), ("const", c, dtype)), ("ge", ("const", c, dtype), ("col", 0))):
                    vectors = [ops.Vector.flat(v, np.ones(n, dtype=bool) if mode == "bitmap" else None)]
                    with pytest.raises(capi.B200Error) as e:
                        run_filter(ctx, None, n, pred, [("col", 0)], vectors=vectors)
                    assert e.value.code == capi.ERR_INVALID


@pytest.mark.parametrize("bitmap", [False, True])
def test_filter_mixed_type_comparison_rejected(ctx, bitmap):
    """A comparison between operands of different types is rejected whatever the path: the tile path used to compare
    UINT8 `< INT64 -5` as signed 64-bit (no row), the interpreter in the column's unsigned type (every row)."""
    n = 5000
    u = (np.arange(n) % 256).astype(np.uint8)
    i = np.arange(n, dtype=np.int32)
    for cols, pred in [([(u, None)], ("lt", ("col", 0), ("const", -5, np.int64))),
                       ([(u, None)], ("gt", ("const", -5, np.int64), ("col", 0))),
                       ([(i, None)], ("eq", ("col", 0), ("const", 7, np.int64))),
                       ([(u, None), (i, None)], ("lt", ("col", 0), ("col", 1))),
                       ([(i, None)], ("distinct", ("col", 0), ("const", 7, np.int16)))]:
        vectors = [ops.Vector.flat(v, np.ones(n, dtype=bool) if bitmap else None) for v, _ in cols]
        with pytest.raises(capi.B200Error) as e:
            run_filter(ctx, None, n, pred, [("col", 0)], vectors=vectors)
        assert e.value.code == capi.ERR_INVALID, pred


def q(v, p):
    """the value at quantile p of column v, as a Python int"""
    s = np.sort(v[:: max(1, len(v) // 4096)])
    return int(s[min(len(s) - 1, int(p * len(s)))])


# columns of the AND-tree test: (dtype, value range)
TREE_COLS = [np.int8, np.uint16, np.int32, np.int64, np.uint8, np.uint32, np.uint64]


def expr_nodes(t):
    return 1 + sum(expr_nodes(c) for c in t[1:] if isinstance(c, tuple)) if t[0] not in ("col", "const") else 1


def tree_preds(cols):
    """AND trees of 1 to 6 `col CMP const` terms over columns of mixed width (one column used twice), each term keeping
    most rows; -> [(predicate, distinct predicate column widths)]"""
    c = lambda i: ("col", i)  # noqa: E731
    k = lambda i, p: ("const", q(cols[i][0], p), TREE_COLS[i])  # noqa: E731

    def conj(*terms):
        t = terms[0]
        for x in terms[1:]:
            t = ("and", t, x)
        return t

    return [
        (("lt", c(2), k(2, 0.6)), [4]),
        (conj(("gt", c(0), k(0, 0.1)), ("le", c(4), k(4, 0.9))), [1, 1]),
        (conj(("ge", c(1), k(1, 0.05)), ("lt", c(1), k(1, 0.95)), ("ne", c(0), k(0, 0.5))), [2, 1]),
        (conj(("gt", c(2), k(2, 0.1)), ("lt", k(5, 0.1), c(5)), ("ge", c(0), k(0, 0.05)), ("ne", c(4), k(4, 0.3))),
         [4, 4, 1, 1]),
        (conj(("le", c(3), k(3, 0.9)), ("gt", c(6), k(6, 0.1)), ("ge", k(2, 0.95), c(2)), ("lt", c(1), k(1, 0.9)),
              ("ne", c(5), k(5, 0.5))), [8, 8, 4, 2, 4]),
        (conj(("gt", c(3), k(3, 0.05)), ("le", c(6), k(6, 0.95)), ("lt", c(2), k(2, 0.9)), ("ge", c(1), k(1, 0.1)),
              ("gt", k(0, 0.95), c(0)), ("ne", c(3), k(3, 0.5))), [8, 8, 4, 2, 1]),
    ]


@pytest.mark.parametrize("n", [1, 31, 2047, 2048, 2049, 4095, 4097, 8191, 8193, 6_000_001])
def test_filter_and_trees(ctx, monkeypatch, n):
    """1..6-term AND trees over columns of mixed width and signedness, at sizes around the 2048-row tile and the 4 K /
    8 K super-tiles, and 6 M rows (every CTA of the mask kernel walks several super-tiles): two-pass TMA kernels,
    the fused single-pass kernel, and the interpreter (all-valid bitmaps) against the oracle."""
    rng = np.random.default_rng(n)
    cols = []
    for dt in TREE_COLS:
        info = np.iinfo(dt)
        cols.append((rng.integers(info.min, info.max, size=n, endpoint=True, dtype=dt), None))
    for pred, widths in tree_preds(cols):
        # a 6-term tree is 23 expression nodes: room for one projection under the 24-node limit
        projs = [("col", 0), ("col", 1), ("col", 2)] if expr_nodes(pred) + 3 <= 24 else [("col", 0)]
        for mode in ("tile", "fused", "bitmap"):
            if mode == "fused":
                monkeypatch.setenv("B200_FILTER_FUSED", "1")
            else:
                monkeypatch.delenv("B200_FILTER_FUSED", raising=False)
            with kernel_trace() as names:
                count = check_filter(ctx, cols, n, pred, projs, bitmap=mode == "bitmap")
            if mode == "tile":
                assert_ran(names, mask_tile_kernel(widths))
                if count:
                    assert_ran(names, "compact_tile_kernel")
                assert_not_ran(names, "filter_mask_kernel", "compact_kernel", "filter_fused_tile_kernel")
            elif mode == "fused":
                assert_ran(names, "filter_fused_tile_kernel")
                assert_not_ran(names, "filter_mask_kernel", "filter_mask_tile_kernel", "compact_kernel")
            else:
                assert_ran(names, "filter_mask_kernel")
                assert_not_ran(names, "filter_mask_tile_kernel", "compact_tile_kernel", "filter_fused_tile_kernel")


PROJ_DTYPES = [np.uint8, np.int16, np.uint32, np.int64, np.int8, np.uint16, np.int32, np.uint64,
               np.uint8, np.int16, np.uint32, np.int64]


@pytest.mark.parametrize("nproj", [1, 2, 5, 12])
def test_filter_projection_widths(ctx, monkeypatch, nproj):
    """1..12 projected columns of every width through the TMA compaction and the fused kernel's shared-memory
    compaction.  Twelve columns do not fit the fused kernel's stages: B200_FILTER_FUSED then takes the two-pass path."""
    rng = np.random.default_rng(100 + nproj)
    n = 100_003
    cols = [(rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, size=n, endpoint=True, dtype=dt), None)
            for dt in PROJ_DTYPES]
    pred = ("lt", ("col", 2), ("const", q(cols[2][0], 0.7), np.uint32))
    projs = [("col", j) for j in range(nproj)]
    for fused in (False, True):
        if fused:
            monkeypatch.setenv("B200_FILTER_FUSED", "1")
        else:
            monkeypatch.delenv("B200_FILTER_FUSED", raising=False)
        with kernel_trace() as names:
            check_filter(ctx, cols, n, pred, projs)
        if fused and nproj < 12:
            assert_ran(names, "filter_fused_tile_kernel")
            assert_not_ran(names, "filter_mask_tile_kernel", "filter_mask_kernel", "compact_kernel")
        else:
            assert_ran(names, mask_tile_kernel([4]), "compact_tile_kernel")
            assert_not_ran(names, "filter_fused_tile_kernel", "filter_mask_kernel", "compact_kernel")


def test_filter_unaligned_input_falls_back(ctx, monkeypatch):
    """a column that does not start on a 16-byte boundary (an offset view) cannot be staged by TMA: the predicate on it
    runs in the interpreter, its projection in the generic compaction, and the answer is unchanged"""
    import torch

    rng = np.random.default_rng(77)
    n = 50_001
    a = rng.integers(-1000, 1000, size=n + 1).astype(np.int32)
    b = rng.integers(-2 ** 62, 2 ** 62, size=n).astype(np.int64)
    ta = torch.from_numpy(a).cuda()
    tb = torch.from_numpy(b).cuda()
    va = ta[1:]                                # 4 bytes past an aligned allocation
    assert va.data_ptr() % 16 != 0 and tb.data_ptr() % 16 == 0
    cols = [(a[1:], None), (b, None)]
    for fused in (False, True):
        if fused:
            monkeypatch.setenv("B200_FILTER_FUSED", "1")
        else:
            monkeypatch.delenv("B200_FILTER_FUSED", raising=False)
        for pred, projs, kernels in [
                (("lt", ("col", 0), ("const", 100, np.int32)), [("col", 1)], ["filter_mask_kernel", "compact_tile_kernel"]),
                (("gt", ("col", 1), ("const", 0, np.int64)), [("col", 0), ("col", 1)],
                 [mask_tile_kernel([8]), "compact_kernel<false>"])]:
            batch = ops.Batch.wrap(ctx, [(va.data_ptr(), capi.INT32), (tb.data_ptr(), capi.INT64)], n, keepalive=[ta, tb])
            e = ops.Expr()
            root = build_expr(e, pred, [capi.INT32, capi.INT64])
            proots = [build_expr(e, p, [capi.INT32, capi.INT64]) for p in projs]
            with kernel_trace() as names:
                out, count, sel, mask = ops.FilterProject(ctx, e, root, proots).execute(batch, want_sel=True, want_mask=True)
            exp_sel, keep = P.filter_select(pred, cols, n)
            assert count == len(exp_sel)
            np.testing.assert_array_equal(sel, exp_sel)
            np.testing.assert_array_equal(capi.valid_from_words(mask, n), keep)
            for (v, _), p in zip(out.download_all(), projs):
                np.testing.assert_array_equal(v, cols[p[1]][0][exp_sel])
            assert_ran(names, *kernels)
            assert_not_ran(names, "filter_fused_tile_kernel")


# ------------------------------------------------------------------ high-cardinality aggregate
def fetch(batch):
    """finalize()'s columns as raw arrays: INT128 -> object array of Python ints (vectorised), others as stored"""
    out = []
    for c, (v, valid) in enumerate(_download_raw(batch)):
        out.append((v, valid))
    return out


def _download_raw(batch):
    import ctypes as C
    n = batch.nrows
    res = []
    for c in range(batch.ncols):
        info = batch.column_info(c)
        raw = np.zeros(2 * n if info.type == capi.INT128 else n,
                       dtype=np.uint64 if info.type == capi.INT128 else capi.DTYPE_OF_TYPE[info.type])
        words = np.zeros(max(1, (n + 63) // 64), dtype=np.uint64)
        capi.check(capi.lib().b200_batch_download(batch.ctx.handle, batch.handle, c,
                                                  C.c_void_p(raw.ctypes.data) if n else None,
                                                  C.c_void_p(words.ctypes.data) if n else None))
        valid = capi.valid_from_words(words, n) if n else np.zeros(0, dtype=bool)
        if info.type == capi.INT128:
            raw = raw[0::2].astype(object) + raw[1::2].view(np.int64).astype(object) * (1 << 64)
        res.append((raw, valid))
    return res


def exact_sums(gid, ng, v, valid):
    """per-group sums of 64-bit integers, exact: 32-bit halves summed by bincount (every partial sum an integer below
    2^53, so the float64 accumulation is exact), recombined as Python ints"""
    if v.dtype == np.int64:
        hi, lo = v >> 32, v & 0xFFFFFFFF
    else:
        hi, lo = v >> np.uint64(32), v & np.uint64(0xFFFFFFFF)
    w = np.ones(len(v)) if valid is None else valid.astype(np.float64)
    H = np.bincount(gid, weights=hi.astype(np.float64) * w, minlength=ng)
    L = np.bincount(gid, weights=lo.astype(np.float64) * w, minlength=ng)
    return H.astype(np.int64).astype(object) * (1 << 32) + L.astype(np.int64).astype(object)


def hc_keys(kw, gid):
    """distinct key tuples per group id, packed into 1, 2 or 3 words (+ the NULL-flag byte)"""
    g = gid.astype(np.int64)
    if kw == 1:
        return [(g * 7 - 1_000_000).astype(np.int32)]
    if kw == 2:
        return [g * 1_000_003 - 2 ** 40]
    return [(g >> 10) * 3 - 2 ** 62, (g & 1023) * 5 + 2 ** 40]


def hc_inputs(rng, nin, n):
    """INT64 / UINT64 columns alternately, full range, with +-2^63 and 2^64-1 planted"""
    cols = []
    for i in range(nin):
        if i % 2 == 0:
            v = rng.integers(-2 ** 63, 2 ** 63, size=n, dtype=np.int64)
            v[rng.integers(0, n, size=500)] = -2 ** 63
            v[rng.integers(0, n, size=500)] = 2 ** 63 - 1
        else:
            v = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
            v[rng.integers(0, n, size=500)] = np.uint64(2 ** 64 - 1)
            v[rng.integers(0, n, size=500)] = np.uint64(2 ** 63)
        cols.append(v)
    return cols


def hc_descs(nin):
    """SUM / SUM_NO_OVERFLOW / COUNT / AVG of input 0, SUM of every other input, COUNT(*)"""
    d = [(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_SUM_NO_OVERFLOW, capi.INT64, 0), (capi.AGG_COUNT, capi.INT64, 0),
         (capi.AGG_AVG, capi.INT64, 0)]
    for i in range(1, nin):
        d.append((capi.AGG_SUM, capi.INT64 if i % 2 == 0 else capi.UINT64, i))
    d.append((capi.AGG_COUNT_STAR, capi.INT64, -1))
    return d


def hc_sink(ctx, agg, keys, key_valid, inputs, in_valid, n, batches=1):
    bounds = np.linspace(0, n, batches + 1).astype(np.int64)
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        vs = [ops.Vector.flat(k[lo:hi], None if key_valid is None else key_valid[lo:hi]) for k in keys]
        vs += [ops.Vector.flat(v[lo:hi], None if in_valid is None else in_valid[lo:hi]) for v in inputs]
        agg.sink(ops.Batch.upload(ctx, vs, int(hi - lo)), list(range(len(keys))),
                 list(range(len(keys), len(keys) + len(inputs))))


def hc_check(res, kw, gid, G, key_valid, inputs, in_valid):
    """finalize() output against exact numpy references: groups matched through their keys"""
    nk = len(hc_keys(kw, np.zeros(1, dtype=np.int64)))
    g = gid if key_valid is None else np.where(key_valid, gid, G)   # rows with a NULL key form group G
    ng = G + 1
    rows = np.bincount(g, minlength=ng)
    present = np.nonzero(rows)[0]
    kv = res[0][1]
    assert len(kv) == len(present), (len(kv), len(present))
    # the group id of every output row, rebuilt from its key
    if kw == 1:
        out_g = (res[0][0].astype(np.int64) + 1_000_000) // 7
    elif kw == 2:
        out_g = (res[0][0].astype(np.int64) + 2 ** 40) // 1_000_003
    else:
        out_g = ((res[0][0] + 2 ** 62) // 3 << 10) + (res[1][0] - 2 ** 40) // 5
    out_g = np.where(kv, out_g, G)
    assert len(np.unique(out_g)) == len(out_g), "duplicate group in the output"
    np.testing.assert_array_equal(np.sort(out_g), present)
    for j in range(nk):
        assert (res[j][1] == (out_g != G)).all()
    a = nk
    v0 = inputs[0]
    s0 = exact_sums(g, ng, v0, in_valid)[out_g]
    c0 = (rows if in_valid is None else np.bincount(g, weights=in_valid, minlength=ng).astype(np.int64))[out_g]
    has = c0 > 0
    sum_v, sum_ok = res[a]
    np.testing.assert_array_equal(sum_ok, has)
    assert (sum_v[has] == s0[has]).all(), "SUM(int64) differs"
    nov, nov_ok = res[a + 1]
    wrapped = np.array([(int(x) + 2 ** 63) % 2 ** 64 - 2 ** 63 for x in s0], dtype=np.int64)
    np.testing.assert_array_equal(nov_ok, has)
    np.testing.assert_array_equal(nov.view(np.int64)[has], wrapped[has])
    np.testing.assert_array_equal(res[a + 2][0].view(np.int64), c0)               # COUNT(x)
    avg, avg_ok = res[a + 3]
    np.testing.assert_array_equal(avg_ok, has)
    exp_avg = np.array([int(s) / int(c) if c else 0.0 for s, c in zip(s0, c0)])  # Python int / int: correctly rounded
    np.testing.assert_allclose(avg[has], exp_avg[has], rtol=1e-15, atol=0)
    for i in range(1, len(inputs)):
        s = exact_sums(g, ng, inputs[i], in_valid)[out_g]
        v, ok = res[a + 3 + i]
        np.testing.assert_array_equal(ok, has)
        assert (v[has] == s[has]).all(), f"SUM of input {i} differs"
    np.testing.assert_array_equal(res[-1][0].view(np.int64), rows[out_g])          # COUNT(*)


def hc_run(ctx, kw, nin, n, G, seed, batches=1, key_nulls=False, input_nulls=False):
    rng = np.random.default_rng(seed)
    gid = rng.integers(0, G, size=n)
    keys = hc_keys(kw, gid)
    key_valid = rng.random(n) > 0.05 if key_nulls else None
    inputs = hc_inputs(rng, nin, n)
    in_valid = rng.random(n) > 0.2 if input_nulls else None
    agg = ops.HashAggregate(ctx, [capi.TYPE_OF_DTYPE[k.dtype] for k in keys], hc_descs(nin))
    with kernel_trace() as names:
        hc_sink(ctx, agg, keys, key_valid, inputs, in_valid, n, batches)
        res = _download_raw(agg.finalize())
    hc_check(res, kw, gid, G, key_valid, inputs, in_valid)
    agg.close()
    return names


def nin_template(nin):
    return 1 if nin <= 1 else 2 if nin <= 2 else 4 if nin <= 4 else 8


@pytest.mark.parametrize("knob", [None, "B200_HC_TILE", "B200_HC_GENERIC"])
@pytest.mark.parametrize("kw,nin", [(1, 1), (2, 2), (3, 3), (1, 5), (2, 8)])
def test_hc_kernels(ctx, monkeypatch, knob, kw, nin):
    """600 K rows in 200 K groups (the adaptation probe picks the HC table; its groups are absorbed into it) with 1- 2-
    and 3-word keys and 1..8 INT64 / UINT64 inputs at +-2^63 and 2^64-1: the direct kernel (no knob), the staged
    kernel (B200_HC_TILE, up to 4 inputs, beyond that the generic one) and the generic kernel (B200_HC_GENERIC) on the
    same data; finalize reads the HC table directly.  (3-word keys go to the HC table from the first row: there is no
    probe table to absorb.)"""
    if knob:
        monkeypatch.setenv(knob, "1")
    names = hc_run(ctx, kw, nin, 600_000, 200_000, seed=kw * 10 + nin)
    if knob is None:
        want = f"agg_hc_direct_kernel<{kw}, {nin_template(nin)}>"
    elif knob == "B200_HC_TILE" and nin <= 4:
        want = f"agg_hc_simple_kernel<{kw}>"
    else:
        want = f"agg_hc_kernel<{kw}, false>"
    assert_ran(names, want, f"agg_hc_finalize_kernel<{kw}>", "hc_count_kernel")
    if kw < 3:
        assert_ran(names, f"agg_hc_absorb_kernel<{kw}>")
    others = {"agg_hc_direct_kernel", "agg_hc_simple_kernel", "agg_hc_kernel"} - {want.split("<")[0]}
    assert_not_ran(names, *others, "agg_hc_flush_kernel")


@pytest.mark.parametrize("kw,key_nulls", [(1, True), (3, False), (2, True)])
def test_hc_nullable(ctx, kw, key_nulls):
    """nullable inputs (cnt[i] arrays) and nullable keys (a NULL group) take the generic staged kernel"""
    names = hc_run(ctx, kw, 2, 600_000, 200_000, seed=50 + kw, key_nulls=key_nulls, input_nulls=True)
    assert_ran(names, f"agg_hc_kernel<{kw}, false>", f"agg_hc_finalize_kernel<{kw}>")
    assert_not_ran(names, "agg_hc_direct_kernel", "agg_hc_simple_kernel")


def test_hc_growth_batches(ctx):
    """3 M rows in three batches over 2 M possible groups: the table starts at 1 M slots, rows that find it full are
    deferred and replayed after it doubles (rehash, count rebalance), later batches sink into the grown table"""
    names = hc_run(ctx, 2, 2, 3_000_000, 2_000_000, seed=7, batches=3)
    assert_ran(names, "agg_hc_direct_kernel<2, 2>", "agg_hc_rehash_kernel<2>", "agg_hc_rows_kernel<2>",
               "hc_spread_count_kernel")


def test_hc_dictionary_keys(ctx):
    """a key column the TMA front end cannot stage (a dictionary vector) with a cardinality hint: the HC table from
    the first row, sunk by the row kernel"""
    rng = np.random.default_rng(91)
    n, G = 400_000, 50_000
    dict_keys = np.arange(G, dtype=np.int32) * 7 - 1_000_000
    gid = rng.integers(0, G, size=n)
    inputs = hc_inputs(rng, 1, n)
    agg = ops.HashAggregate(ctx, [capi.INT32], hc_descs(1), expected_groups=G)
    with kernel_trace() as names:
        b = ops.Batch.upload(ctx, [ops.Vector.dictionary(dict_keys, gid.astype(np.uint32)), ops.Vector.flat(inputs[0])], n)
        agg.sink(b, [0], [1])
        res = _download_raw(agg.finalize())
    hc_check(res, 1, gid, G, None, inputs, None)
    agg.close()
    assert_ran(names, "agg_hc_rows_kernel<1>", "agg_hc_finalize_kernel<1>")
    assert_not_ran(names, "agg_hc_direct_kernel", "agg_hc_kernel")


@pytest.mark.parametrize("kw", [1, 3])
def test_hc_export_combine(ctx, kw):
    """partial tables in the HC path exported (the HC table is first flushed into the generic table) and merged:
    export_states -> combine_states and export_packed -> combine_packed on one GPU equal one table over all rows"""
    import torch

    rng = np.random.default_rng(200 + kw)
    n, G, nin = 800_000, 150_000, 2
    gid = rng.integers(0, G, size=n)
    keys = hc_keys(kw, gid)
    inputs = hc_inputs(rng, nin, n)
    key_types = [capi.TYPE_OF_DTYPE[k.dtype] for k in keys]
    half = n // 2
    for packed in (False, True):
        parts = []
        with kernel_trace() as names:
            for lo, hi in ((0, half), (half, n)):
                a = ops.HashAggregate(ctx, key_types, hc_descs(nin))
                hc_sink(ctx, a, [k[lo:hi] for k in keys], None, [v[lo:hi] for v in inputs], None, hi - lo)
                parts.append(a)
            final = ops.HashAggregate(ctx, key_types, hc_descs(nin))
            for a in parts:
                if packed:
                    words = a.packed_words(G)
                    buf = torch.empty(words, dtype=torch.int64, device="cuda:0")
                    a.export_packed(buf.data_ptr(), G)
                    final.combine_packed(buf.data_ptr(), 1, G)
                    ctx.sync()
                else:
                    final.combine_states(a.export_states())
            res = _download_raw(final.finalize())
        hc_check(res, kw, gid, G, None, inputs, None)
        assert_ran(names, f"agg_hc_direct_kernel<{kw}, 2>", f"agg_hc_flush_kernel<{kw}>")
        for a in parts + [final]:
            a.close()


# ------------------------------------------------------------------ join, lean probe
EMPTY_BITS = np.uint64(1 << 63)   # the open-addressing table's empty-slot key: INT64_MIN, or 2^63 as UBIGINT
PAYLOADS = {"none": [], "u8": [np.uint8], "i16": [np.int16], "u8u8": [np.uint8, np.uint8], "i32": [np.int32]}


def join_data(rng, dtype, dense, nb, npb):
    """unique build keys and probe keys of which ~70 % hit.  dense: a compact key range (for UBIGINT one that straddles
    2^63); otherwise keys spread over all 64 bits with the empty-slot key on both sides."""
    if dense:
        start = EMPTY_BITS - np.uint64(nb // 2) if dtype == np.uint64 else np.uint64(2 ** 64 - nb)   # -nb for BIGINT
        bits = start + rng.permutation(2 * nb)[:nb].astype(np.uint64)
        miss = np.uint64(3 * nb)               # past the key range
    else:
        bits = np.unique(np.concatenate([rng.integers(0, 2 ** 64, size=nb, dtype=np.uint64), [EMPTY_BITS]]))
        rng.shuffle(bits)
        miss = None
    pbits = bits[rng.integers(0, len(bits), size=npb)]
    m = rng.random(npb) < 0.3
    pbits[m] = pbits[m] + miss if dense else pbits[m] ^ np.uint64(0x5555_0000_5555)
    if not dense:
        pbits[rng.integers(0, npb, size=1000)] = EMPTY_BITS
    return bits.view(dtype), pbits.view(dtype)


def check_join(ctx, bk, pk, nlhs, payload, rng):
    nb, npb = len(bk), len(pk)
    bp = [rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, size=nb, endpoint=True, dtype=dt) for dt in PAYLOADS[payload]]
    lhs = [rng.integers(-2 ** 63, 2 ** 63, size=npb, dtype=np.int64) for _ in range(nlhs)]
    (res, sel, count), names = traced(lambda: run_join(ctx, "inner", [(bk, None)], [(p, None) for p in bp],
                                                       [(pk, None)], [(v, None) for v in lhs], nb, npb))
    order = np.argsort(bk, kind="stable")
    pos = np.minimum(np.searchsorted(bk[order], pk), nb - 1)
    hit = bk[order][pos] == pk
    brow = order[pos]
    assert count == int(hit.sum())
    np.testing.assert_array_equal(np.sort(sel), np.nonzero(hit)[0])
    for j in range(nlhs):
        np.testing.assert_array_equal(res[j][0], lhs[j][sel])
    for p in range(len(bp)):
        np.testing.assert_array_equal(res[nlhs + p][0], bp[p][brow[sel]])
    return names


@pytest.mark.parametrize("rows", [8, 4])
@pytest.mark.parametrize("dense", [True, False])
@pytest.mark.parametrize("dtype", [np.int64, np.uint64])
def test_join_lean_probe(ctx, monkeypatch, rows, dense, dtype):
    """the lean probe (INNER join, unique BIGINT / UBIGINT build keys, payload inline or none) with 8 and 4 rows per
    thread, on the dense table and on open addressing (EMPTY_KEY on both sides goes to the side slot), 0..4 lhs
    columns, payloads none / 1 byte / 2 bytes / two 1-byte; 1.1 M probe rows span several waves of the grid.  With 8
    rows per thread, 3 or 4 lhs columns do not fit two stages in 110 KB and the round-1 lean kernel takes them."""
    if rows == 4:
        monkeypatch.setenv("B200_JOIN_ROWS", "4")
    if not dense:
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(rows * 4 + dense * 2 + (dtype == np.uint64))
    bk, pk = join_data(rng, dtype, dense, 300_000, 1_100_000)
    for nlhs, payload in [(0, "none"), (1, "u8"), (2, "i16"), (3, "u8u8"), (4, "u8"), (2, "none"), (0, "u8u8")]:
        names = check_join(ctx, bk, pk, nlhs, payload, rng)
        fits = (2 if rows == 8 else 3) * rows * 256 * 8 * (1 + nlhs) <= 110 * 1024
        if fits:
            assert_ran(names, f"join_probe_lean2_kernel<{nlhs}, {rows}, {'true' if dense else 'false'}>")
            assert_not_ran(names, "join_probe_tile_kernel")
        else:
            assert_ran(names, "join_probe_tile_kernel<true, true>")
            assert_not_ran(names, "join_probe_lean2_kernel")


@pytest.mark.parametrize("dense", [True, False])
def test_join_lean1_and_control(ctx, monkeypatch, dense):
    """B200_JOIN_LEAN1 runs the round-1 lean kernel; a 4-byte payload is not inline in the lean sense, so the same keys
    take the FAST8 non-lean kernel"""
    if not dense:
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(300 + dense)
    bk, pk = join_data(rng, np.int64, dense, 300_000, 1_100_000)
    monkeypatch.setenv("B200_JOIN_LEAN1", "1")
    names = check_join(ctx, bk, pk, 2, "u8", rng)
    assert_ran(names, "join_probe_tile_kernel<true, true>")
    assert_not_ran(names, "join_probe_lean2_kernel")
    monkeypatch.delenv("B200_JOIN_LEAN1")
    names = check_join(ctx, bk, pk, 2, "i32", rng)
    assert_ran(names, "join_probe_tile_kernel<true, false>")
    assert_not_ran(names, "join_probe_lean2_kernel", "join_probe_tile_kernel<true, true>")

