"""MARK hash joins (large IN lists, IN subqueries outside a plain conjunct, NOT IN) through B200HashJoin against the stock
operator, in the way of tests/test_gpu_duckdb_operators.py: every query runs in one connection twice through the
decorated plan and once with B200_DISABLE=1, and the results must agree bit for bit, NULL marks included.  The EXPLAIN
of the decorated plan must show B200_HASH_JOIN over a MARK join - without "(host)" on a GPU.

Probe sizes sit at the 128 K-row batch boundary (B200_PROBE_BATCH) with threads=1, so one worker sees every chunk and
the batch arithmetic is exact; a threads=4 pass covers the per-worker result buffers.  Without a CUDA device the
decorator forwards to the stock operator and the plumbing variants check the "(host)" plan and the same results."""
import ctypes as C
import os

import pytest

from test_gpu_duckdb_operators import EXT, JOIN_OPTIMIZERS, PROBE_BATCH, _compare, _Env

PROBE_SIZES = [PROBE_BATCH - 1, PROBE_BATCH, PROBE_BATCH + 1]

TABLES = [
    # k: ~1/3 of the rows fall in 0 .. 299, NULL one row in 53; kb the same as BIGINT; kd DOUBLE with -0.0 and NaN
    *[f"""CREATE TABLE mp_{n} AS SELECT i AS pid,
            CASE WHEN i % 53 = 11 THEN NULL ELSE ((i * 2654435761) % 900)::INTEGER END AS k,
            CASE WHEN i % 53 = 11 THEN NULL ELSE ((i * 2654435761) % 900)::BIGINT + 4294967296 END AS kb,
            CASE WHEN i % 61 = 5 THEN 'nan'::DOUBLE WHEN i % 67 = 6 THEN -0.0
                 ELSE ((i * 40503) % 600)::DOUBLE / 4 END AS kd,
            'row-' || i AS s
        FROM range({n}) r(i)""" for n in PROBE_SIZES],
    # subquery build sides: mb_k without NULL, mb_kn with one NULL key
    "CREATE TABLE mb AS SELECT (3 * i)::INTEGER AS k, CASE WHEN i = 17 THEN NULL ELSE (5 * i)::INTEGER END AS kn, "
    "(i * 0.5)::DOUBLE AS kd, i % 4 AS f FROM range(100) r(i)",
    # TPC-H Q16's NOT IN shape on numeric columns: partsupp x supplier (s_flag marks the complaint suppliers)
    "CREATE TABLE partsupp AS SELECT i // 4 AS ps_partkey, ((i * 7919) % 10000)::INTEGER AS ps_suppkey "
    "FROM range(400000) r(i)",
    "CREATE TABLE supplier AS SELECT i::INTEGER AS s_suppkey, (i % 37 = 3)::INTEGER AS s_flag FROM range(10000) r(i)",
]

# 43 constants: above the rewrite threshold.  The lists sit in the select list: in a WHERE clause the filter
# pushdown hands them to the scan, and no join is planned
IN_LIST = ", ".join(str(v) for v in range(0, 300, 7))
IN_LIST_NULL = IN_LIST + ", NULL"
IN_LIST_BIG = ", ".join(str(4294967296 + v) for v in range(0, 300, 11))
IN_LIST_DOUBLE = "0.0, 'nan'::DOUBLE, 1.25, 2.5, 10.0, 100.75, 149.75, -3.0"


def _cases():
    cases = []
    for n in PROBE_SIZES:
        p = f"mp_{n}"
        cases += [
            (f"in-list-{n}", 1, f"SELECT pid, k IN ({IN_LIST}) AS m FROM {p} ORDER BY pid"),
            (f"in-list-null-{n}", 1, f"SELECT pid, k IN ({IN_LIST_NULL}) AS m FROM {p} ORDER BY pid"),
            (f"not-in-list-{n}", 1, f"SELECT pid, s, k NOT IN ({IN_LIST}) AS m FROM {p} ORDER BY pid"),
            (f"in-subquery-select-{n}", 1, f"SELECT pid, k IN (SELECT k FROM mb) AS m FROM {p} ORDER BY pid"),
        ]
    p = "mp_131073"
    cases += [
        ("in-list-bigint", 1, f"SELECT pid, kb IN ({IN_LIST_BIG}) AS m FROM {p} ORDER BY pid"),
        ("in-list-double", 1, f"SELECT pid, kd IN ({IN_LIST_DOUBLE}) AS m FROM {p} ORDER BY pid"),
        ("not-in-list-null", 1, f"SELECT pid, k NOT IN ({IN_LIST_NULL}) AS m FROM {p} ORDER BY pid"),
        ("in-subquery-null-build", 1, f"SELECT pid, k IN (SELECT kn FROM mb) AS m FROM {p} ORDER BY pid"),
        ("in-subquery-or", 1, f"SELECT pid, s FROM {p} WHERE k IN (SELECT k FROM mb WHERE f = 1) OR pid % 3 = 0 "
                              "ORDER BY pid"),
        ("not-in-subquery-null-build", 1, f"SELECT pid FROM {p} WHERE k NOT IN (SELECT kn FROM mb) ORDER BY pid"),
        ("in-subquery-empty-build", 1, f"SELECT pid, k IN (SELECT k FROM mb WHERE f = 7) AS m FROM {p} ORDER BY pid"),
        ("q16-not-in", 1, "SELECT ps_partkey, ps_suppkey FROM partsupp WHERE ps_suppkey NOT IN "
                          "(SELECT s_suppkey FROM supplier WHERE s_flag = 1) ORDER BY ps_partkey, ps_suppkey"),
    ]
    for t in (1, 4):
        cases += [
            (f"in-list-t{t}-1m", t, f"SELECT pid, k IN ({IN_LIST_NULL}) AS m FROM {p} ORDER BY pid"),
            (f"q16-not-in-t{t}", t, "SELECT ps_partkey, ps_suppkey FROM partsupp WHERE ps_suppkey NOT IN "
                                    "(SELECT s_suppkey FROM supplier WHERE s_flag = 1) ORDER BY ps_partkey, ps_suppkey"),
        ]
    return cases


CASES = _cases()


def _serve(pipe):
    """the child process of db(): owns the connection and runs _compare requests until it receives None"""
    from oracle import duckdb_ref as R

    R.lib()
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
        except Exception as e:
            pipe.send(("assert" if isinstance(e, AssertionError) else "error", f"{type(e).__name__}: {e}"))
    con.close()
    pipe.close()


@pytest.fixture(scope="module")
def db():
    """(pipe to a connection in a child process, has_device), as in test_gpu_duckdb_operators.py"""
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


def _mark_case(db, device, case):
    name, threads, sql = case
    pipe, has_device = db
    if device:
        assert has_device, "the gpu tests need a CUDA device"
    elif has_device:
        pytest.skip("with a CUDA device the decorator runs on it: the gpu-marked variant runs this case")
    settings = {"threads": threads, "disabled_optimizers": JOIN_OPTIMIZERS, "perfect_ht_threshold": 0}
    planned = "B200_HASH_JOIN" if device else "B200_HASH_JOIN(host)"
    pipe.send((settings, sql, {}, planned, "B200_HASH_JOIN(host)" if device else None))
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(f"{result}\nquery: {sql}")
    plan, exp = result
    assert "MARK" in plan, plan
    rows = len(exp[0].values)
    if " AS m FROM mp_" in sql:
        # a mark in the select list: one result row per probe row, NULL marks where the shape has them
        assert rows == int(sql.split(" AS m FROM mp_")[1].split()[0]), (name, rows)
        m = exp[-1]
        has_null = m.valid is not None and not m.valid.all()
        if "null" in name:
            assert has_null, name                        # a NULL in the list / on the build side
        if "empty" in name:
            assert not has_null and not m.values.any(), name   # FALSE for every row, NULL keys too
    else:
        assert rows > 0 or "null" in name, (name, rows)  # NOT IN with a NULL on the build side keeps no row


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mark_join_matches_the_stock_operator(db, case):
    _mark_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mark_join_on_the_gpu_matches_the_stock_operator(db, case):
    _mark_case(db, True, case)
