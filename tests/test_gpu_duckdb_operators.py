"""The DuckDB operators of integration/ (B200HashJoin, B200HashAggregate, B200Filter, B200BatchedFilter) against the
stock operators, at the batch, morsel and chunk boundaries of the binding.

Every query runs in ONE connection over the same tables: twice through the decorated plan and once with B200_DISABLE=1,
which the optimizer hook reads at plan time and which leaves the stock plan in place.  The EXPLAIN of the decorated
plan must name the operator under test - without "(host)" on a GPU, so a query cannot pass by falling back to the stock
operator - and both decorated runs must return exactly the rows of the stock run: same order (every query sorts on a
unique key), same types, same validity, same values bit for bit.  SUM / AVG over DOUBLE only see dyadic values whose
partial sums are exact, so the summation order cannot change a bit; integer AVG uses the same long-double formula on
both sides.

The tables are built in SQL over range(n) with integer hashing, so every size is exact.  The boundary cases run with
threads=1, so one worker sees every chunk in table order and the batch arithmetic is deterministic:
  - hash join: the probe side is buffered until B200_PROBE_BATCH = 131 072 rows (64 full chunks) are there; results
    larger than the batch go through the B200_ERR_CAPACITY -> count -> re-probe path; results are emitted grouped by
    input chunk; the build side is flushed to the device every B200_MORSEL_ROWS = 1 048 576 rows;
  - hash aggregate: morsels of 1 048 576 rows cycle through a ring of two pinned buffers, Combine sinks the last two;
    the result is converted chunk by chunk (HUGEINT / BIGINT sums, integer AVG with the DECIMAL scale, NULLs);
  - filter: batches of B200_FILTER_BATCH rows (below one chunk, 0 included, one chunk per kernel call).
A second pass at threads=4 covers the pooled contexts, the per-worker rings and the parallel Combine.

Without a CUDA device every decorator forwards to the stock operator: the plumbing tests run the same queries, check
the "(host)" decorator is planned and the results are equal.  With a device they skip; the gpu-marked tests run them."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = os.path.join(ROOT, "integration", "_build", "libb200_duckdb.so")

PROBE_BATCH = 128 * 1024      # B200_PROBE_BATCH, integration/b200_join.cpp
MORSEL_ROWS = 1 << 20         # B200_MORSEL_ROWS, integration/b200_binding.hpp
PROBE_SIZES = [PROBE_BATCH - 1, PROBE_BATCH, PROBE_BATCH + 1, 2 * PROBE_BATCH + 5, 1000003]
AGG_ROWS = 5000000
FILTER_ROWS = 1000003

JOIN_OPTIMIZERS = "build_side_probe_side,join_order"   # keep the sides as written: the right side is the build side
# without aggregate_function_rewriter, AVG stays an aggregate (the rewriter plans avg(x) as sum(x) / count(x))
AGG_OPTIMIZERS = "statistics_propagation,aggregate_function_rewriter"
FILTER_OPTIMIZERS = "filter_pushdown,statistics_propagation"  # keep the predicate in a LogicalFilter


# ---------------------------------------------------------------------------------------------------------- tables
def _probe_table(n):
    # key: ~30 % of the rows hit an even build key below 200 000; every fourth run of 10 000 rows (about five whole
    # chunks) holds keys no build row has; one row in 101 has a NULL key
    return f"""CREATE TABLE jp_{n} AS SELECT pid, key::INTEGER AS ki, (key + 1099511627776)::BIGINT AS kb,
                   DATE '1970-01-01' + key::INTEGER AS kd, ((key % 65536) - 32768)::SMALLINT AS ks,
                   CASE WHEN pid % 101 = 7 THEN NULL ELSE (2 * ((pid * 2654435761) % 40000))::INTEGER END AS kh,
                   CASE WHEN pid % 101 = 7 THEN NULL ELSE ((pid * 2654435761) % 80000)::INTEGER END AS km,
                   CASE WHEN pid % 101 = 7 THEN NULL ELSE ((pid * 2654435761) % 10000000)::INTEGER END AS kg,
                   'probe-side-row-' || pid AS s
               FROM (SELECT i AS pid, CASE WHEN i % 101 = 7 THEN NULL
                                           WHEN (i // 10000) % 4 = 3 THEN 1000000000 + i
                                           ELSE (i * 2654435761) % 250000 END AS key FROM range({n}) r(i))"""


TABLES = [
    # build side: unique even keys 0, 2, .., 199 998 (NULL one row in 97), in four key types; payloads of 1, 2, 4, 8
    # bytes with NULLs. ks repeats every 32 768 rows, so the SMALLINT join also has duplicate build keys
    """CREATE TABLE jb AS SELECT i AS bid,
           CASE WHEN i % 97 = 5 THEN NULL ELSE (2 * i)::INTEGER END AS ki,
           CASE WHEN i % 97 = 5 THEN NULL ELSE (2 * i + 1099511627776)::BIGINT END AS kb,
           CASE WHEN i % 97 = 5 THEN NULL ELSE DATE '1970-01-01' + (2 * i)::INTEGER END AS kd,
           CASE WHEN i % 97 = 5 THEN NULL ELSE (((2 * i) % 65536) - 32768)::SMALLINT END AS ks,
           CASE WHEN i % 5 = 1 THEN NULL ELSE (i % 251 - 125)::TINYINT END AS p1,
           CASE WHEN i % 7 = 2 THEN NULL ELSE (i % 60000 - 30000)::SMALLINT END AS p2,
           CASE WHEN i % 11 = 3 THEN NULL ELSE (i * 37 - 1000000)::INTEGER END AS p4,
           CASE WHEN i % 13 = 4 THEN NULL ELSE i * 1000000007 - 1125899906842624 END AS p8,
           CASE WHEN i % 17 = 6 THEN NULL ELSE i / 4 END AS pd
       FROM range(100000) r(i)""",
    # every key 0, 2, .., 79 998 five times
    """CREATE TABLE jb5 AS SELECT i AS bid, CASE WHEN i % 89 = 3 THEN NULL ELSE (2 * (i % 40000))::INTEGER END AS k,
           CASE WHEN i % 7 = 2 THEN NULL ELSE (i % 60000 - 30000)::SMALLINT END AS p2
       FROM range(200000) r(i)""",
    # 2.5 M build rows: two full build morsels and a partial one on one worker
    """CREATE TABLE jbig AS SELECT i AS bid, CASE WHEN i % 89 = 3 THEN NULL ELSE (3 * i)::INTEGER END AS k,
           CASE WHEN i % 13 = 4 THEN NULL ELSE i * 1000000007 END AS p8
       FROM range(2500000) r(i)""",
] + [_probe_table(n) for n in PROBE_SIZES] + [
    # 5 M aggregate input rows; g<m> has m groups and a NULL group ((i * 2654435761) % m is a bijection on each run of
    # m rows: every group occurs)
    f"""CREATE TABLE ag AS SELECT
           CASE WHEN i % 1009 = 0 THEN NULL ELSE (i * 2654435761) % 5 END AS g5,
           CASE WHEN i % 1009 = 0 THEN NULL ELSE ((i * 2654435761) % 35)::INTEGER END AS g35,
           CASE WHEN i % 1009 = 0 THEN NULL ELSE ((i * 2654435761) % 600)::SMALLINT END AS g600,
           CASE WHEN i % 1009 = 0 THEN NULL ELSE (i * 2654435761) % 200000 END AS g200000,
           CASE WHEN i % 1009 = 0 THEN NULL ELSE ((i * 2654435761) % 1500000)::INTEGER END AS g1500000,
           CASE WHEN i % 13 = 0 THEN NULL ELSE ((i * 7919) % 2000001 - 1000000)::INTEGER END AS vi,
           CASE WHEN i % 17 = 0 THEN NULL ELSE (i * 1000003) % 2000000000000 - 1000000000000 END AS vb,
           -- near +-2^62: the group sums leave the int64 range (HUGEINT results)
           CASE WHEN i % 5 < 3 THEN 4611686018427387904 - i % 1000 ELSE -4611686018427387904 + i % 777 END AS vh,
           CASE WHEN i % 11 = 0 THEN NULL ELSE (((i * 37) % 100000000 - 50000000) / 100)::DECIMAL(15,2) END AS vd,
           -- dyadic: multiples of 2^-10 below 32 in magnitude, every partial sum of 5 M of them is exact
           CASE WHEN i % 19 = 0 THEN NULL ELSE ((i * 40503) % 65536 - 32768)::DOUBLE / 1024 END AS vf,
           CASE WHEN i % 100003 = 7 THEN 'nan'::DOUBLE WHEN i % 100003 = 11 THEN 'inf'::DOUBLE
                WHEN i % 100003 = 13 THEN '-inf'::DOUBLE WHEN i % 29 = 0 THEN NULL
                ELSE ((i * 31337) % 1000003)::DOUBLE / 8 - 60000 END AS vm,
           CASE WHEN i % 23 = 0 THEN NULL ELSE DATE '1992-01-01' + ((i * 7) % 3000)::INTEGER END AS vt
       FROM range({AGG_ROWS}) r(i)""",
    # filter input: fr alternates in runs of 1 500 rows, fn is NULL in every third row
    f"""CREATE TABLE ft AS SELECT i::INTEGER AS fi, ((i * 40503) % 65536)::DOUBLE / 8 AS fd, 'f' || i AS fs,
           ((i // 1500) % 2)::INTEGER AS fr, CASE WHEN i % 3 = 0 THEN NULL ELSE ((i * 7919) % 1000)::INTEGER END AS fn
       FROM range({FILTER_ROWS}) r(i)""",
]


class _Env:
    """set environment variables for a block (the optimizer hook and the operators read them at plan time)"""

    def __init__(self, env):
        self.env, self.saved = env, {}

    def __enter__(self):
        for k, v in self.env.items():
            self.saved[k] = os.environ.get(k)
            os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _plan(con, sql, env):
    with _Env(env):
        return "\n".join(str(r[-1]) for r in con.fetchall("EXPLAIN " + sql))


def _assert_same(got, exp, what, by_value=()):
    """equal types, validity and values, floats bit for bit (any NaN equals any NaN).  Float columns named in
    `by_value` compare by value (-0.0 equals 0.0): float group keys, which hold the first value a group saw, and MIN /
    MAX over groups that hold both zeros"""
    assert [c.name for c in got] == [c.name for c in exp], what
    assert [(c.type_id, c.scale) for c in got] == [(c.type_id, c.scale) for c in exp], what
    for g, e in zip(got, exp):
        n = len(e.values)
        assert len(g.values) == n, (what, g.name, "row count", len(g.values), n)
        gv = np.ones(n, bool) if g.valid is None else g.valid
        ev = np.ones(n, bool) if e.valid is None else e.valid
        bad = np.flatnonzero(gv != ev)
        assert bad.size == 0, (what, g.name, "NULL at different rows", bad[:10])
        a, b = g.values[ev], e.values[ev]
        if a.dtype.kind == "f":
            nan = np.isnan(b)
            bits = np.dtype(f"u{a.dtype.itemsize}")    # FLOAT results are 4 bytes wide
            same = (a == b) if g.name in by_value else (a.view(bits) == b.view(bits))
            diff = (np.isnan(a) != nan) | (~nan & ~same)
        elif a.dtype == object:
            diff = np.array([x != y for x, y in zip(a, b)], dtype=bool)
        else:
            diff = a != b
        bad = np.flatnonzero(diff)
        assert bad.size == 0, (what, g.name, "values differ at", np.flatnonzero(ev)[bad[:10]], a[bad[:5]], b[bad[:5]])


def _compare(con, settings, sql, env, planned, not_planned, by_value=()):
    """in the child: the plan must name `planned` and not `not_planned`; then two decorated runs against one stock run
    (`by_value`: see _assert_same).  -> (plan, the stock result without its HUGEINT / VARCHAR values, which are slow to
    pickle)"""
    for k, v in settings.items():
        con.execute(f"SET {k}='{v}'" if isinstance(v, str) else f"SET {k}={v}")
    plan = _plan(con, sql, env)
    assert planned in plan and (not not_planned or not_planned not in plan), plan
    with _Env(env):
        got = [con.execute(sql), con.execute(sql)]
    stock = {"B200_DISABLE": "1"}
    assert "B200_" not in _plan(con, sql, stock)
    with _Env(stock):
        exp = con.execute(sql)
    for i, g in enumerate(got):
        _assert_same(g, exp, f"run {i + 1}: {sql}", by_value)
    for c in exp:
        if c.values.dtype == object:
            c.values = None
    return plan, exp


def _serve(pipe):
    """the child process of db(): owns the connection and runs _compare requests until it receives None"""
    from oracle import duckdb_ref as R

    R.lib()  # the reference library first, so the binding resolves its DuckDB symbols against the same copy
    ext = C.CDLL(EXT, mode=C.RTLD_GLOBAL)
    ext.b200_duckdb_register.argtypes = [C.c_void_p]
    con = R.Connection(threads=4)
    assert ext.b200_duckdb_register(con.db) == 0
    with _Env({"B200_DISABLE": "1"}):
        for sql in TABLES:
            con.execute(sql)
    pipe.send(ext.b200_device_count() > 0)
    while True:
        request = pipe.recv()
        if request is None:
            break
        try:
            pipe.send(("ok", _compare(con, *request)))
        except Exception as e:  # a failed assertion or query fails the test that sent it
            pipe.send(("assert" if isinstance(e, AssertionError) else "error", f"{type(e).__name__}: {e}"))
    con.close()
    pipe.close()


@pytest.fixture(scope="module")
def db():
    """(pipe to the connection, has_device).  The connection lives in a child process: after a few minutes of DuckDB
    queries on the device, a process's CUPTI activity tracing stopped recording kernels (H100, torch 2.11), and the
    kernel-path tests that run later in the same pytest process need it.  The child exits when the module is done."""
    import multiprocessing

    from oracle import duckdb_ref as R

    if not R.available() or not os.path.exists(EXT):
        pytest.skip("needs oracle/_ref/libduckdb_ref.so and integration/_build/libb200_duckdb.so (built by build())")
    spawn = multiprocessing.get_context("spawn")
    parent, child = spawn.Pipe()
    proc = spawn.Process(target=_serve, args=(child,), daemon=True)
    proc.start()
    child.close()
    try:
        has_device = parent.recv()
        yield parent, has_device
        parent.send(None)
        proc.join(timeout=120)
    finally:
        if proc.is_alive():
            proc.terminate()
            proc.join()
        parent.close()


# ------------------------------------------------------------------------------------------------------ comparison
def _check(db, device, sql, operator, settings, env=None):
    """run `sql` twice through the decorated plan and once on the stock plan, in the child; returns the stock result
    (numeric columns only) and the plan"""
    pipe, has_device = db
    if device:
        assert has_device, "the gpu tests need a CUDA device"
    elif has_device:
        pytest.skip("with a CUDA device the decorators run on it: the gpu-marked variant runs this case")
    pipe.send((settings, sql, env or {}, operator if device else operator + "(host)", operator + "(host)" if device else None))
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(f"{result}\nquery: {sql}")
    plan, exp = result
    return exp, plan


# ------------------------------------------------------------------------------------------------------- hash join
def _join_sql(kind, probe, build, key, build_key=None, payload=("bid", "p1", "p2", "p4", "p8", "pd"), probe_cols=("pid",)):
    lhs = ", ".join("p." + c for c in probe_cols)
    if kind in ("SEMI", "ANTI"):
        return f"SELECT {lhs} FROM {probe} p {kind} JOIN {build} b ON p.{key} = b.{build_key or key} ORDER BY p.pid"
    rhs = ", ".join("b." + c for c in payload)
    return (f"SELECT {lhs}, {rhs} FROM {probe} p {kind} JOIN {build} b ON p.{key} = b.{build_key or key} "
            f"ORDER BY p.pid, b.bid")


JOIN_KINDS = ["INNER", "LEFT", "SEMI", "ANTI"]
EMPTY_BUILD = "(SELECT * FROM jb WHERE bid % 2 = 2)"    # no row, and nothing the optimizer can prove
JOIN_CASES = []
for _n in PROBE_SIZES:                                   # batch boundaries: 64 full chunks = one batch
    for _kind in JOIN_KINDS:
        JOIN_CASES.append((f"batch-{_n}-{_kind}-t1", 1, _join_sql(_kind, f"jp_{_n}", "jb", "ki")))
for _kind in JOIN_KINDS:                                 # pooled contexts, one batch ring per worker
    JOIN_CASES.append((f"batch-1000003-{_kind}-t4", 4, _join_sql(_kind, "jp_1000003", "jb", "ki")))
for _key in ["kb", "kd", "ks"]:                          # key types (INTEGER is above), NULL keys on both sides
    for _kind in JOIN_KINDS:
        JOIN_CASES.append((f"key-{_key}-{_kind}", 1, _join_sql(_kind, "jp_131073", "jb", _key)))
for _kind in ["INNER", "LEFT"]:                          # a VARCHAR probe column, carried by slicing
    JOIN_CASES.append((f"varchar-{_kind}", 1, _join_sql(_kind, "jp_262149", "jb", "ki", probe_cols=("pid", "s"))))
for _t in [1, 4]:                                        # results of ~5x the batch: capacity retry
    JOIN_CASES.append((f"capacity-INNER-t{_t}", _t, _join_sql("INNER", "jp_262149", "jb5", "kh", "k", ("bid", "p2"))))
    JOIN_CASES.append((f"capacity-LEFT-t{_t}", _t, _join_sql("LEFT", "jp_262149", "jb5", "km", "k", ("bid", "p2"))))
for _kind in ["INNER", "LEFT", "ANTI"]:                  # partial input chunks (and runs of chunks without a match)
    JOIN_CASES.append((f"partial-chunks-{_kind}", 1,
                       _join_sql(_kind, "(SELECT * FROM jp_1000003 WHERE pid % 7 <> 3)", "jb", "ki")))
for _kind in JOIN_KINDS:                                 # empty sides
    JOIN_CASES.append((f"empty-build-{_kind}", 1, _join_sql(_kind, "jp_131073", EMPTY_BUILD, "ki")))
    JOIN_CASES.append((f"empty-probe-{_kind}", 1,
                       _join_sql(_kind, "(SELECT * FROM jp_131073 WHERE pid % 2 = 2)", "jb", "ki")))
for _kind, _t in [("INNER", 1), ("LEFT", 1), ("INNER", 4)]:   # several build morsels per worker
    JOIN_CASES.append((f"build-morsels-{_kind}-t{_t}", _t, _join_sql(_kind, "jp_1000003", "jbig", "kg", "k", ("bid", "p8"))))


def _join_case(db, device, case):
    name, threads, sql = case
    settings = {"threads": threads, "disabled_optimizers": JOIN_OPTIMIZERS, "perfect_ht_threshold": 0}
    exp, _ = _check(db, device, sql, "B200_HASH_JOIN", settings)
    rows = len(exp[0].values)
    # the shapes reach what they are named for
    if name.startswith("empty-build"):
        assert rows == (131073 if name.endswith(("LEFT", "ANTI")) else 0), (name, rows)  # every probe row, or none
    if name.startswith("empty-probe"):
        assert rows == 0, (name, rows)
    if name.startswith("capacity-INNER"):
        assert rows > 4 * 262149 * 0.9, rows
    if name.startswith("capacity-LEFT"):
        assert rows > 2 * 262149, rows


@pytest.mark.parametrize("case", JOIN_CASES, ids=[c[0] for c in JOIN_CASES])
def test_hash_join_matches_the_stock_operator(db, case):
    _join_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", JOIN_CASES, ids=[c[0] for c in JOIN_CASES])
def test_hash_join_on_the_gpu_matches_the_stock_operator(db, case):
    _join_case(db, True, case)


# -------------------------------------------------------------------------------------------------- hash aggregate
AGG_SELECTS = {
    "int": "count(*), count(vi), sum(vi), min(vi), max(vi), avg(vi), count(vb), sum(vb), min(vb), max(vb), avg(vb)",
    "wide": "count(*), sum(vh), avg(vh), min(vh), max(vh), count(vd), sum(vd), avg(vd), min(vd), max(vd)",
    "float-date": "count(*), count(vf), sum(vf), avg(vf), count(vm), min(vm), max(vm), count(vt), min(vt), max(vt)",
}
# default optimizer settings: sum over INTEGER and DECIMAL(15,2) inputs plans as sum_no_overflow, avg as sum / count
STATS_SELECT = "count(*), sum(vi), avg(vi), min(vi), max(vi), count(vd), sum(vd), avg(vd), min(vd), max(vd), sum(vf)"
GROUP_COUNTS = [5, 35, 600, 200000, 1500000]
AGG_CASES = []
for _g in GROUP_COUNTS:
    for _t in [1, 4]:
        for _what, _sel in AGG_SELECTS.items():
            AGG_CASES.append((f"{_what}-g{_g}-t{_t}", _t, _g, AGG_OPTIMIZERS, _sel))
        AGG_CASES.append((f"stats-g{_g}-t{_t}", _t, _g, "", STATS_SELECT))


def _agg_case(db, device, case):
    from oracle import duckdb_ref as R

    name, threads, groups, optimizers, select = case
    sql = f"SELECT g{groups}, {select} FROM ag GROUP BY g{groups} ORDER BY g{groups}"
    settings = {"threads": threads, "disabled_optimizers": optimizers, "perfect_ht_threshold": 0}
    exp, plan = _check(db, device, sql, "B200_HASH_GROUP_BY", settings)
    if optimizers:
        assert plan.count("avg(") == select.count("avg("), plan   # integer AVG: sum and count, divided on the host
    if name.startswith("stats"):
        # statistics rule out an int64 overflow: the int64-state variant is planned; its result type stays HUGEINT /
        # DECIMAL(38,2) in this DuckDB, and the decorator must return the same type
        assert plan.count("sum_no_overflow") == 2, plan
        assert [(c.type_id, c.scale) for c in (exp[2], exp[7])] == [(R.T_HUGEINT, 0), (R.T_DECIMAL, 2)]
    # every group once, and the NULL group
    keys = exp[0]
    assert len(keys.values) == groups + 1 and keys.valid is not None and not keys.valid[-1]
    assert np.array_equal(keys.values[:-1].astype(np.int64), np.arange(groups)), name
    assert int(exp[1].values.sum()) == AGG_ROWS


@pytest.mark.parametrize("case", AGG_CASES, ids=[c[0] for c in AGG_CASES])
def test_hash_aggregate_matches_the_stock_operator(db, case):
    _agg_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", AGG_CASES, ids=[c[0] for c in AGG_CASES])
def test_hash_aggregate_on_the_gpu_matches_the_stock_operator(db, case):
    _agg_case(db, True, case)


# ---------------------------------------------------------------------------------------------------------- filter
FILTER_PREDICATES = {
    "all": "fd <> 0.3",        # 0.3 lies inside the column's range, but no fd (a multiple of 1/8) equals it
    "none": "fd = 0.3",
    "runs": "fr = 0",          # alternating runs of 1 500 rows
    "nullable": "fn < 500",
}
FILTER_BATCHES = ["0", "1", "2047", "2048", "2049", "5000", None]
FILTER_CASES = []
for _scan in [False, True]:
    for _b in FILTER_BATCHES:
        for _p in FILTER_PREDICATES:
            FILTER_CASES.append((f"{'scan-' if _scan else ''}batch-{_b or 'default'}-{_p}", _scan, _b, _p))


def _filter_case(db, device, case):
    name, scan, batch, pred = case
    sql = f"SELECT fi, fd, fs FROM ft WHERE {FILTER_PREDICATES[pred]} ORDER BY fi"
    env = {"B200_SCAN_FILTERS": "1"} if scan else {}
    if batch is not None:
        env["B200_FILTER_BATCH"] = batch
    settings = {"threads": 1, "disabled_optimizers": "" if scan else FILTER_OPTIMIZERS, "perfect_ht_threshold": 0}
    exp, _ = _check(db, device, sql, "B200_FILTER", settings, env)
    rows = len(exp[0].values)
    assert (rows == FILTER_ROWS) if pred == "all" else (rows == 0) if pred == "none" else (0 < rows < FILTER_ROWS)


@pytest.mark.parametrize("case", FILTER_CASES, ids=[c[0] for c in FILTER_CASES])
def test_filter_matches_the_stock_operator(db, case):
    _filter_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FILTER_CASES, ids=[c[0] for c in FILTER_CASES])
def test_filter_on_the_gpu_matches_the_stock_operator(db, case):
    _filter_case(db, True, case)
