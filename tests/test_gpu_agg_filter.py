"""Filtered aggregates (b200_agg_create_filtered, FILTER (WHERE ...)) through operators.HashAggregate(filters=...),
checked against exact references and the kernel trace.

The rule is DuckDB's: every row creates its group, and a filtered aggregate is updated only with the rows where its
BOOLEAN filter column is TRUE (NULL and FALSE skip it, physical_hash_aggregate.cpp:361-404).  For the functions the
device supports that is "the input is NULL where the filter is not TRUE", so the reference here is the unfiltered
reference of tests/test_gpu_agg_kernel_paths.py over inputs with that validity; count(*) FILTER (f) is COUNT over the
column f with validity "f valid and nonzero".  Integer sums are exact Python ints, integer AVG is long double(sum) /
count like the library's finalize, MIN / MAX are bit-exact except that float MIN / MAX compare +-0.0 by value.

The fold runs once per sink call (agg_filter_fold_kernel) and hands the sink nullable inputs.  The register path
(FASTREG) and the private paths (PRIV / WPRIV) take no nullable input, so at their group counts a filtered aggregate
runs the shared-memory FAST and MID kernels; the high-cardinality table runs its generic kernel (its simple and direct
kernels take no validity either), and with B200_AGG_NO_HC=1 the generic table runs agg_sink_kernel."""
import os
import time
import traceback

import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran
from test_gpu_agg_kernel_paths import (FUNC, PROBE, assert_same, canon, fetch_groups, planted, reference,
                                       traced_window)

pytestmark = pytest.mark.gpu

# kernel of agg_filter.cu -> the tests here that assert it ran
KERNEL_CASES = {
    "agg_filter_fold_kernel": ["test_every_function_and_filter_kind", "test_groups_and_state_sharing",
                               "test_vector_shapes", "test_sink_paths", "test_export_combine_states",
                               "test_export_combine_packed",
           "test_all_minus_one_is_the_unfiltered_aggregate"],
}
KERNEL_EXCLUDED = {}


# ------------------------------------------------------------------ the worker process
# The kernel trace loses kernels once the process's first profiler session lies more than about 10 s back, and records
# none after about a minute (DESIGN.md §9): a module that traced in the pytest process would push every later traced
# module past that.  So the cases below run, and trace, in spawned worker processes of their own, each replaced once it
# has traced for WORKER_SECONDS; the tests send the cases there and check the kernel names they return.
def _serve(pipe):
    import torch

    torch.cuda.set_device(0)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    while True:
        request = pipe.recv()
        if request is None:
            break
        name, args, env = request
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            pipe.send(("ok", globals()[name](ctx, *args)))
        except Exception as e:
            pipe.send(("assert" if isinstance(e, AssertionError) else "error", traceback.format_exc()))
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    ctx.close()
    pipe.close()


WORKER_SECONDS = 10   # a worker that has traced for this long is replaced before the next case


class _Worker:
    def __init__(self):
        import multiprocessing

        spawn = multiprocessing.get_context("spawn")
        self.pipe, child = spawn.Pipe()
        self.proc = spawn.Process(target=_serve, args=(child,), daemon=True)
        self.proc.start()
        child.close()
        self.started = None   # set by the first case: the worker's first profiler session

    def close(self):
        try:
            self.pipe.send(None)
            self.proc.join(timeout=120)
        finally:
            if self.proc.is_alive():
                self.proc.terminate()
                self.proc.join()
            self.pipe.close()


@pytest.fixture(scope="module")
def cases():
    """-> run(case name, *args, env={}): the case's result, from a worker process that has traced for less than
    WORKER_SECONDS when the case starts"""
    current = [None]

    def run(name, *args, env=None):
        w = current[0]
        if w is None or (w.started is not None and time.monotonic() - w.started > WORKER_SECONDS):
            if w is not None:
                w.close()
            w = current[0] = _Worker()
        if w.started is None:
            w.started = time.monotonic()
        w.pipe.send((name, args, env or {}))
        status, result = w.pipe.recv()
        if status != "ok":
            raise (AssertionError if status == "assert" else RuntimeError)(f"in the worker:\n{result}")
        return result

    try:
        yield run
    finally:
        if current[0] is not None:
            current[0].close()


# ------------------------------------------------------------------ the reference
def passes(filt):
    """rows where a filter column (values, valid | None) is TRUE: valid and a nonzero byte"""
    v, valid = filt
    p = np.asarray(v).view(np.uint8) != 0
    return p if valid is None else p & valid


def unfiltered_problem(inputs, filters, aggs):
    """aggs: [(func, input | -1, filter | -1)] -> (inputs, aggs) of the unfiltered problem with the same answer"""
    eff, out, at = [], [], {}
    for f, i, k in aggs:
        if f == "count_star" and k < 0:
            out.append(("count_star", -1))
            continue
        key = ("star", k) if f == "count_star" else (i, k)
        if key not in at:
            if f == "count_star":
                eff.append((np.asarray(filters[k][0]).view(np.uint8), passes(filters[k])))
            else:
                v, valid = inputs[i]
                if k >= 0:
                    valid = passes(filters[k]) if valid is None else valid & passes(filters[k])
                eff.append((v, valid))
            at[key] = len(eff) - 1
        out.append(("count" if f == "count_star" else f, at[key]))
    return eff, out


def float_minmax(gid, ng, v, valid, func):
    """MIN / MAX of floats per group as DuckDB orders them (NaN above everything); None without a valid value"""
    ok = np.ones(len(v), dtype=bool) if valid is None else valid
    nan = np.isnan(v)
    has = np.bincount(gid[ok], minlength=ng) > 0
    has_nan = np.bincount(gid[ok & nan], minlength=ng) > 0
    has_num = np.bincount(gid[ok & ~nan], minlength=ng) > 0
    sel = ok & ~nan
    if func == "min":
        out = np.full(ng, np.inf, dtype=v.dtype)
        np.minimum.at(out, gid[sel], v[sel])
        return [None if not has[g] else float(out[g]) if has_num[g] else float("nan") for g in range(ng)]
    out = np.full(ng, -np.inf, dtype=v.dtype)
    np.maximum.at(out, gid[sel], v[sel])
    return [None if not has[g] else float("nan") if has_nan[g] else float(out[g]) for g in range(ng)]


def expected(keys, gid, ng, eff, eaggs):
    """reference() for the integer / float-sum aggregates, float_minmax for float MIN / MAX"""
    isfmm = [f in ("min", "max") and np.asarray(eff[i][0]).dtype.kind == "f" for f, i in eaggs]
    plain = [a for a, m in zip(eaggs, isfmm) if not m]
    exp = reference(keys, gid, ng, eff, plain)
    first = np.full(ng, -1, dtype=np.int64)
    first[gid[::-1]] = np.arange(len(gid) - 1, -1, -1)
    fm = {a: float_minmax(gid, ng, np.asarray(eff[a[1]][0]), eff[a[1]][1], a[0]) for a, m in zip(eaggs, isfmm) if m}
    out = {}
    for g in np.nonzero(first >= 0)[0]:
        r = first[g]
        key = tuple(canon(k[r]) if kv is None or kv[r] else None for k, kv in keys)
        it = iter(exp[key])
        out[key] = [fm[a][g] if m else next(it) for a, m in zip(eaggs, isfmm)]
    return out


# ------------------------------------------------------------------ running an aggregate
def dictionary_of(v, valid):
    """the same logical column as a dictionary vector: reversed, behind three unused NULL entries"""
    n = len(v)
    d = np.concatenate([np.zeros(3, dtype=v.dtype), v[::-1]])
    dv = np.concatenate([np.zeros(3, dtype=bool), np.ones(n, dtype=bool) if valid is None else valid[::-1]])
    return ops.Vector.dictionary(d, (3 + n - 1 - np.arange(n)).astype(np.uint32), dv)


def vector(v, valid, form, lo, hi):
    if form == "constant":
        assert (v[lo:hi] == v[lo]).all() and (valid is None or (valid[lo:hi] == valid[lo]).all())
        return ops.Vector.constant(v[lo], v.dtype, is_null=valid is not None and not valid[lo])
    if form == "dictionary":
        return dictionary_of(v[lo:hi], None if valid is None else valid[lo:hi])
    return ops.Vector.flat(v[lo:hi], None if valid is None else valid[lo:hi])


def descs(inputs, filters, aggs):
    return [(FUNC[f], capi.TYPE_OF_DTYPE[np.asarray(inputs[i][0]).dtype] if i >= 0 else capi.INT64, i)
            for f, i, _ in aggs], [-1 if k < 0 else len(inputs) + k for _, _, k in aggs]


def sink_batches(ctx, agg, keys, inputs, filters, bounds, forms=None):
    """input_cols = [inputs..., filters...]; forms: {column of input_cols: "flat" | "constant" | "dictionary"}"""
    forms = forms or {}
    cols = list(inputs) + list(filters)
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        vs = [ops.Vector.flat(k[lo:hi], None if kv is None else kv[lo:hi]) for k, kv in keys]
        vs += [vector(v, valid, forms.get(c, "flat"), lo, hi) for c, (v, valid) in enumerate(cols)]
        agg.sink(ops.Batch.upload(ctx, vs, int(hi - lo)), list(range(len(keys))),
                 list(range(len(keys), len(keys) + len(cols))))


def run_filtered(ctx, keys, gid, ng, inputs, filters, aggs, bounds=None, forms=None, expected_groups=0):
    """sink + finalize in the kernel trace, checked against the reference; -> kernel names"""
    bounds = [0, len(gid)] if bounds is None else bounds
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]
    d, f = descs(inputs, filters, aggs)

    def run():
        agg = ops.HashAggregate(ctx, key_types, d, expected_groups, filters=f)
        sink_batches(ctx, agg, keys, inputs, filters, bounds, forms)
        out = fetch_groups(agg.finalize(), len(keys), len(aggs))
        agg.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel", "agg_filter_fold_kernel"])
    eff, eaggs = unfiltered_problem(inputs, filters, aggs)
    assert_same(got, expected(keys, gid, ng, eff, eaggs), eaggs, eff)
    return names, got


def filter_column(rng, n, kind, null_frac=0.2):
    """a BOOL filter column: all_true, all_false, mixed (TRUE bytes of 1, 2 and 255), null_rows (mixed with NULLs)"""
    if kind == "all_true":
        return np.ones(n, dtype=bool), None
    if kind == "all_false":
        return np.zeros(n, dtype=bool), None
    b = rng.choice(np.array([0, 0, 1, 2, 255], dtype=np.uint8), size=n).view(np.bool_)
    return b, (rng.random(n) > null_frac if kind == "null_rows" else None)


def values(rng, dtype, n):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = (rng.standard_normal(n) * 1e3).astype(dt)
        v[rng.integers(0, n, size=5)] = -0.0
        return v
    if dt.itemsize == 8:
        return planted(rng, dtype, n, -2 ** 62 if dt.kind == "i" else 0, 2 ** 62)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, size=n, endpoint=True).astype(dt)


# ------------------------------------------------------------------ functions x filters
DTYPES = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint32, np.uint64, np.float32, np.float64]


def case_every_function_and_filter_kind(ctx, dtype, kind):
    """COUNT_STAR, COUNT, SUM, SUM_NO_OVERFLOW (integers), MIN, MAX, AVG under one filter, over a nullable input, next
    to the same functions unfiltered; three sink calls"""
    rng = np.random.default_rng(DTYPES.index(dtype) * 10 + len(kind))
    n, ng = 60_001, 20
    gid = rng.integers(0, ng, size=n)
    keys = [((gid * 3 - 20).astype(np.int16), None)]
    x = values(rng, dtype, n)
    inputs = [(x, rng.random(n) > 0.1)]
    filters = [filter_column(rng, n, kind)]
    fns = ["count", "sum", "min", "max", "avg"] + (["sum_no_overflow"] if np.dtype(dtype).kind != "f" else [])
    aggs = [("count_star", -1, 0)] + [(f, 0, 0) for f in fns] + [("count_star", -1, -1)] + [(f, 0, -1) for f in fns]
    names, got = run_filtered(ctx, keys, gid, ng, inputs, filters, aggs, bounds=[0, 7, n // 2, n])
    assert len(got) == ng
    if kind == "all_false":
        assert all(v[0] == 0 and v[1] == 0 and all(x is None for x in v[2:len(fns) + 1]) for v in got.values())
    return names


def case_groups_and_state_sharing(ctx):
    """groups whose every row fails the filter (FALSE in one, NULL in another) exist with COUNT 0 and NULL SUM / MIN
    / MAX / AVG; sum(x), sum(x) FILTER (p), sum(x) FILTER (q) and avg(x) FILTER (p) keep three sums"""
    rng = np.random.default_rng(5)
    n, ng = 200_003, 50
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.int32) * 1000, None)]
    x = rng.integers(-2 ** 40, 2 ** 40, size=n, dtype=np.int64)
    p, pv = filter_column(rng, n, "null_rows")
    p[gid == 0] = False
    pv[gid == 1] = False
    q, _ = filter_column(rng, n, "mixed")
    inputs = [(x, None)]
    filters = [(p, pv), (q, None)]
    aggs = [("sum", 0, -1), ("sum", 0, 0), ("sum", 0, 1), ("avg", 0, 0), ("count", 0, 0), ("min", 0, 0),
            ("max", 0, 1), ("count_star", -1, 0), ("count_star", -1, 1), ("count_star", -1, -1)]
    names, got = run_filtered(ctx, keys, gid, ng, inputs, filters, aggs, bounds=[0, n // 3, n])
    for g in (0, 1):
        r = got[(g * 1000,)]
        assert r[0] is not None and r[1] is None and r[2] is not None and r[3] is None and r[4] == 0, r
        assert r[5] is None and r[7] == 0 and r[9] > 0, r
    r = got[(2000,)]
    assert len({r[0], r[1], r[2]}) == 3, r
    return names


# ------------------------------------------------------------------ vector forms
SHAPES = {
    "input-constant": ({0: "constant"}, "mixed"),
    "input-constant-null": ({0: "constant"}, "mixed"),
    "input-dictionary": ({0: "dictionary"}, "null_rows"),
    "filter-dictionary": ({1: "dictionary"}, "null_rows"),
    "both-dictionary": ({0: "dictionary", 1: "dictionary"}, "null_rows"),
    "filter-constant-true": ({1: "constant"}, "all_true"),
    "filter-constant-false": ({1: "constant"}, "all_false"),
    "filter-constant-null": ({1: "constant"}, "constant_null"),
    "dictionary-input-constant-filter": ({0: "dictionary", 1: "constant"}, "all_true"),
}


def case_vector_shapes(ctx, shape):
    """FLAT, CONSTANT and DICTIONARY inputs and filters (dictionary validity is indexed by dictionary position), with
    a FLAT input over the same column unfiltered; integer and double inputs"""
    rng = np.random.default_rng(len(shape))
    forms, kind = SHAPES[shape]
    n, ng = 30_000, 12
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.uint8), None)]
    x = rng.integers(-2 ** 50, 2 ** 50, size=n, dtype=np.int64)
    xv = rng.random(n) > 0.2
    d = rng.standard_normal(n)
    if forms.get(0) == "constant":
        x, xv = np.full(n, -12345, dtype=np.int64), np.full(n, shape != "input-constant-null")
        d = np.full(n, 2.5)
    if kind == "constant_null":
        filt = (np.ones(n, dtype=bool), np.zeros(n, dtype=bool))
    else:
        filt = filter_column(rng, n, kind)
    inputs = [(x, xv), (d, None)]
    filters = [filt]
    aggs = [("sum", 0, 0), ("count", 0, 0), ("min", 0, 0), ("max", 0, 0), ("avg", 0, 0), ("sum", 1, 0),
            ("max", 1, 0), ("count_star", -1, 0), ("sum", 0, -1), ("count_star", -1, -1)]
    # input_cols = [x, d, filter]: forms name input 0 (x) and the filter (column 2)
    cforms = {0: forms[0]} if 0 in forms else {}
    if 1 in forms:
        cforms[2] = forms[1]
    names, got = run_filtered(ctx, keys, gid, ng, inputs, filters, aggs, bounds=[0, 10_000, n], forms=cforms)
    if kind in ("all_false", "constant_null"):
        assert all(v[1] == 0 and v[0] is None and v[7] == 0 for v in got.values())
    return names


# ------------------------------------------------------------------ sink paths
PATHS = {
    # name: (groups, rows, batch bounds, env, kernel that must run, kernels that must not)
    "fast4": (3, PROBE + 300_001, [0, 100_000, PROBE + 7], {}, "agg_fast_kernel",
              ["agg_fastreg_kernel", "agg_mid_kernel"]),
    "fast": (7, PROBE + 300_001, [0, PROBE - 1], {}, "agg_fast_kernel", ["agg_fastreg_kernel", "agg_mid_kernel"]),
    "priv": (35, 1_000_001, [0, PROBE + 1], {"B200_AGG_NO_WPRIV": "1"}, "agg_mid_kernel",
             ["agg_priv_kernel", "agg_wpriv_kernel"]),
    "wpriv": (35, 1_000_001, [0, PROBE + 1], {"B200_AGG_WPRIV": "1"}, "agg_mid_kernel",
              ["agg_priv_kernel", "agg_wpriv_kernel"]),
    "mid": (300, 1_000_001, [0, 500_000], {}, "agg_mid_kernel", ["agg_priv_kernel", "agg_wpriv_kernel"]),
    "hc": (200_000, 3_500_001, [0, 1_000_003, 1_500_000], {}, "agg_hc_kernel",
           ["agg_hc_simple_kernel", "agg_hc_direct_kernel"]),
    "generic": (200_000, 3_500_001, [0, 1_000_003, 1_500_000], {"B200_AGG_NO_HC": "1"}, "agg_sink_kernel",
                ["agg_hc_kernel", "agg_hc_simple_kernel", "agg_hc_direct_kernel"]),
}


def case_sink_paths(ctx, path):
    """each sink path, chosen by the group count (or its knob), with filtered and unfiltered aggregates over the same
    inputs; batches cross the 256 K-row adaptation probe and the high-cardinality table's 1 M / 2 M-row chunks"""
    ng, n, bounds, env, kernel, absent = PATHS[path]
    assert all(os.environ.get(k) == v for k, v in env.items()), env   # (set by the worker, see cases())
    rng = np.random.default_rng(len(path) * 7)
    gid = rng.integers(0, ng, size=n)
    gid[:ng] = np.arange(ng)
    if ng <= 64:
        keys = [((gid // 5).astype(np.uint8), None), ((gid % 5).astype(np.uint8), None)]
    else:
        keys = [((gid * 7 - 10 ** 6).astype(np.int32), None)]
    x = planted(rng, np.int64, n, -2 ** 39, 2 ** 39)
    y = planted(rng, np.uint64, n, 0, 2 ** 40)
    p = filter_column(rng, n, "null_rows")
    q = filter_column(rng, n, "mixed")
    p[0][gid == 1] = False                                   # group 1 passes no row of p
    inputs = [(x, rng.random(n) > 0.1), (y, None)]
    filters = [p, q]
    aggs = [("sum", 0, 0), ("sum", 0, -1), ("count", 0, 0), ("avg", 0, 1), ("sum", 1, 0), ("sum", 1, -1),
            ("count_star", -1, 1), ("count_star", -1, -1)]
    if path not in ("priv", "wpriv", "hc"):
        aggs += [("min", 0, 0), ("max", 1, 1), ("sum_no_overflow", 0, 1)]
    names, got = run_filtered(ctx, keys, gid, ng, inputs, filters, aggs, bounds=bounds + [n])
    assert len(got) == ng
    assert_not_ran(names, *absent)
    return names


# ------------------------------------------------------------------ no fold without a filter
def case_all_minus_one_is_the_unfiltered_aggregate(ctx):
    """an aggregate without filters launches no fold; b200_agg_create_filtered with every filter -1 gives the same
    result and the same launches as b200_agg_create; a filter on one aggregate leaves the others' results alone"""
    rng = np.random.default_rng(9)
    n, ng = PROBE + 50_001, 6
    gid = rng.integers(0, ng, size=n)
    keys = [(gid.astype(np.uint8), None)]
    x = planted(rng, np.int64, n, -2 ** 39, 2 ** 39)
    inputs = [(x, None)]
    fcol = filter_column(rng, n, "mixed")
    d, _ = descs(inputs, [], [("sum", 0, -1), ("avg", 0, -1), ("count_star", -1, -1)])
    bounds = [0, n // 2, n]

    def run(filters):
        before = ctx.stats()["launches"]
        agg = ops.HashAggregate(ctx, [capi.UINT8], d, 0, filters=filters)
        cols = inputs + ([fcol] if filters and max(filters) >= 0 else [])
        for lo, hi in zip(bounds[:-1], bounds[1:]):
            vs = [ops.Vector.flat(keys[0][0][lo:hi])] + [ops.Vector.flat(v[lo:hi], None if m is None else m[lo:hi])
                                                          for v, m in cols]
            agg.sink(ops.Batch.upload(ctx, vs, hi - lo), [0], list(range(1, len(vs))))
        out = fetch_groups(agg.finalize(), 1, len(d))
        agg.close()
        return out, ctx.stats()["launches"] - before

    (plain, plain_launches), plain_names = traced_window(lambda: run(None), always=["agg_init_kernel"])
    (minus, minus_launches), minus_names = traced_window(lambda: run([-1, -1, -1]), always=["agg_init_kernel"])
    assert plain == minus
    assert plain_launches == minus_launches
    assert sorted(set(plain_names)) == sorted(set(minus_names))
    assert_not_ran(plain_names, "agg_filter_fold_kernel")
    assert_not_ran(minus_names, "agg_filter_fold_kernel")
    (filt, _), filt_names = traced_window(lambda: run([1, -1, -1]),
                                          always=["agg_init_kernel", "agg_filter_fold_kernel"])
    assert_ran(filt_names, "agg_filter_fold_kernel")
    return plain_names, minus_names, filt_names
    assert {k: v[1:] for k, v in filt.items()} == {k: v[1:] for k, v in plain.items()}   # the unfiltered AVG, count(*)


# ------------------------------------------------------------------ export / combine
def combine_case(rng, n, ng):
    gid = rng.integers(0, ng, size=n)
    keys = [((gid // 4).astype(np.uint8), None), ((gid % 4).astype(np.int16), None)]
    x = rng.integers(-2 ** 50, 2 ** 50, size=n, dtype=np.int64)
    d = rng.standard_normal(n)
    inputs = [(x, rng.random(n) > 0.2), (d, None)]
    filters = [filter_column(rng, n, "null_rows"), filter_column(rng, n, "mixed")]
    filters[0][0][gid == 2] = False
    aggs = [("sum", 0, 0), ("sum", 0, -1), ("avg", 0, 1), ("count", 0, 0), ("min", 0, 1), ("max", 1, 0),
            ("sum", 1, 1), ("count_star", -1, 0), ("count_star", -1, -1)]
    return gid, keys, inputs, filters, aggs


def partial_aggregates(ctx, keys, inputs, filters, aggs, parts):
    key_types = [capi.TYPE_OF_DTYPE[np.asarray(k).dtype] for k, _ in keys]
    d, f = descs(inputs, filters, aggs)
    out = []
    for lo, hi in parts:
        a = ops.HashAggregate(ctx, key_types, d, filters=f)
        if hi > lo:
            sink_batches(ctx, a, [(k[lo:hi], None) for k, _ in keys],
                         [(v[lo:hi], None if m is None else m[lo:hi]) for v, m in inputs],
                         [(v[lo:hi], None if m is None else m[lo:hi]) for v, m in filters], [0, hi - lo])
        out.append(a)
    return out, ops.HashAggregate(ctx, key_types, d, filters=f)


def case_export_combine_states(ctx):
    """partial filtered aggregates exported as state columns (one block per (input, filter) pair) and combined into an
    aggregate created with the same descs and filters: equal to one aggregate over all rows"""
    rng = np.random.default_rng(11)
    n, ng = 300_000, 24
    gid, keys, inputs, filters, aggs = combine_case(rng, n, ng)

    def run():
        parts, final = partial_aggregates(ctx, keys, inputs, filters, aggs, [(0, n // 3), (n // 3, n)])
        for a in parts:
            final.combine_states(a.export_states())
            a.close()
        out = fetch_groups(final.finalize(), len(keys), len(aggs))
        final.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel", "agg_filter_fold_kernel"])
    eff, eaggs = unfiltered_problem(inputs, filters, aggs)
    assert_same(got, expected(keys, gid, ng, eff, eaggs), eaggs, eff)
    assert_ran(names, "agg_filter_fold_kernel", "agg_export_kernel", "agg_combine_kernel")
    return names


def case_export_combine_packed(ctx):
    """the packed partial states of three filtered aggregates (one of them empty) in one device buffer, combined"""
    import torch

    rng = np.random.default_rng(12)
    n, ng = 90_000, 24
    gid, keys, inputs, filters, aggs = combine_case(rng, n, ng)
    max_groups = 32

    def run():
        parts, final = partial_aggregates(ctx, keys, inputs, filters, aggs, [(0, n // 3), (n // 3, n // 3),
                                                                             (n // 3, n)])
        words = parts[0].packed_words(max_groups)
        buf = torch.zeros(3 * words, dtype=torch.int64, device="cuda:0")
        for r, a in enumerate(parts):
            a.export_packed(buf.data_ptr() + r * words * 8, max_groups)
        final.combine_packed(buf.data_ptr(), 3, max_groups)
        ctx.sync()
        out = fetch_groups(final.finalize(), len(keys), len(aggs))
        for a in parts + [final]:
            a.close()
        return out

    got, names = traced_window(run, always=["agg_init_kernel", "agg_filter_fold_kernel"])
    eff, eaggs = unfiltered_problem(inputs, filters, aggs)
    assert_same(got, expected(keys, gid, ng, eff, eaggs), eaggs, eff)
    assert_ran(names, "agg_filter_fold_kernel", "agg_export_packed_kernel", "agg_combine_packed_kernel")
    return names


# ------------------------------------------------------------------ sink-time checks
def case_sink_rejects_a_filter_that_is_not_bool(ctx):
    """a filter column of another type, and a column index past the batch, are B200_ERR_INVALID"""
    n = 1000
    k = np.zeros(n, dtype=np.uint8)
    x = np.arange(n, dtype=np.int64)
    agg = ops.HashAggregate(ctx, [capi.UINT8], [(capi.AGG_SUM, capi.INT64, 0)], filters=[1])
    b = ops.Batch.upload(ctx, [ops.Vector.flat(k), ops.Vector.flat(x), ops.Vector.flat(x)], n)
    with pytest.raises(capi.B200Error) as e:
        agg.sink(b, [0], [1, 2])
    assert e.value.code == capi.ERR_INVALID and "B200_BOOL" in str(e.value)
    rc = capi.lib().b200_agg_sink(agg.handle, b.handle, capi.int_array([0]), capi.int_array([1, 3]))
    assert rc == capi.ERR_INVALID
    agg.close()


# ------------------------------------------------------------------ the tests: each runs its case in the worker
@pytest.mark.parametrize("kind", ["all_true", "all_false", "mixed", "null_rows"])
@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_every_function_and_filter_kind(cases, dtype, kind):
    assert_ran(cases("case_every_function_and_filter_kind", dtype, kind), "agg_filter_fold_kernel")


def test_groups_and_state_sharing(cases):
    assert_ran(cases("case_groups_and_state_sharing"), "agg_filter_fold_kernel")


@pytest.mark.parametrize("shape", list(SHAPES))
def test_vector_shapes(cases, shape):
    assert_ran(cases("case_vector_shapes", shape), "agg_filter_fold_kernel")


@pytest.mark.parametrize("path", list(PATHS))
def test_sink_paths(cases, path):
    names = cases("case_sink_paths", path, env=PATHS[path][3])
    assert_ran(names, "agg_filter_fold_kernel", PATHS[path][4])
    assert_not_ran(names, *PATHS[path][5])


def test_all_minus_one_is_the_unfiltered_aggregate(cases):
    plain, minus, filt = cases("case_all_minus_one_is_the_unfiltered_aggregate")
    assert_not_ran(plain, "agg_filter_fold_kernel")
    assert_not_ran(minus, "agg_filter_fold_kernel")
    assert_ran(filt, "agg_filter_fold_kernel")


def test_export_combine_states(cases):
    assert_ran(cases("case_export_combine_states"), "agg_filter_fold_kernel", "agg_export_kernel", "agg_combine_kernel")


def test_export_combine_packed(cases):
    assert_ran(cases("case_export_combine_packed"), "agg_filter_fold_kernel", "agg_export_packed_kernel",
               "agg_combine_packed_kernel")


def test_sink_rejects_a_filter_that_is_not_bool(cases):
    cases("case_sink_rejects_a_filter_that_is_not_bool")
