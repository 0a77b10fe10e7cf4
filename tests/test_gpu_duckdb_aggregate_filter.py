"""B200HashAggregate over filtered aggregates (FILTER (WHERE ...), and the filtered aggregates DuckDB binds a small
PIVOT to) against the stock PhysicalHashAggregate, in the way of tests/test_gpu_duckdb_aggregate_types.py: every
query runs in one connection twice through the decorated plan and once with B200_DISABLE=1, and the results must
agree - same types, same validity, values bit for bit (MIN / MAX over doubles compare +-0.0 by value).

Decorated (the plan must show B200_HASH_GROUP_BY, without "(host)" on a GPU):
  - FILTER on count(*), count, sum, min, max and avg over integer, DECIMAL and double inputs, with predicates that are
    NULL in some rows and predicates that no row of most groups passes, next to unfiltered aggregates over the same
    columns, at 5, 600, 200 000 and 1 500 000 groups, threads 1 and 4 with the rewriter and statistics off (integer AVG
    in the binding), threads 4 with the default settings (sum_no_overflow, avg as sum / count), and the large group
    counts again with B200_AGG_NO_HC=1; 1 600 003 rows cross a 1 M-row morsel;
  - 12 filtered aggregates;
  - PIVOT with and without an IN list, with USING sum(x), count(*) and with the default count(*), grouped by a numeric
    column: DuckDB binds it as one filtered aggregate per pivot value.
Compared only (whatever plan DuckDB picks): count(DISTINCT x) FILTER (WHERE p), which the multi-stage rewriter turns
into an outer aggregate that carries the filter.
Stock (the plan names no B200 operator, the results still agree): a filtered ungrouped aggregate, and a filter in a
list of 13 aggregates.

Without a CUDA device the decorator forwards to the stock operator: the plumbing variants check the "(host)" plans
and the same results.  With a device they skip; the gpu-marked variants run the cases."""
import ctypes as C
import os

import pytest

from test_gpu_duckdb_aggregate_types import _check, _settings
from test_gpu_duckdb_operators import AGG_OPTIMIZERS, EXT, _compare, _Env

ROWS = 1600003
GROUP_COUNTS = [5, 600, 200000, 1500000]
NULL_KEY = f"i % 1009 = 0 AND i >= {GROUP_COUNTS[-1]}"
TABLE = f"""CREATE TABLE tf AS SELECT i AS rid,
    {', '.join(f"CASE WHEN {NULL_KEY} THEN NULL ELSE ((i * 2654435761) % {g})::INTEGER END AS g{g}"
               for g in GROUP_COUNTS)},
    CASE WHEN i % 11 = 0 THEN NULL ELSE ((i * 40503) % 65536 - 32768)::SMALLINT END AS i16,
    CASE WHEN i % 17 = 0 THEN NULL ELSE ((i * 2654435761) % 4294967296 - 2147483648)::INTEGER END AS i32,
    CASE WHEN i % 19 = 0 THEN NULL
         ELSE ((i::HUGEINT * 11400714819323198485) % 18446744073709551616 - 9223372036854775808)::BIGINT END AS i64,
    ((i * 37) % 256)::UTINYINT AS u8,
    CASE WHEN i % 53 = 0 THEN NULL
         ELSE ((i * 2654435761) % 1999999999 - 999999999)::DECIMAL(18,0) * 0.01 END::DECIMAL(9,2) AS d92,
    CASE WHEN i % 67 = 0 THEN NULL WHEN i % 31 = 3 THEN '-0.0'::DOUBLE
         ELSE ((i * 31337) % 1048576 - 524288)::DOUBLE / 4096 END AS f64,
    CASE WHEN i % 7 = 0 THEN NULL ELSE (i * 37) % 3 = 0 END AS p,
    (i % 4)::INTEGER AS pv
FROM range({ROWS}) r(i)"""
FLOAT_MIN_MAX = ("min_f", "max_f")


# ------------------------------------------------------------------------------------------------ child process
def _serve(pipe):
    """the child process of db(): owns the connection and runs _compare requests until it receives None"""
    from oracle import duckdb_ref as R

    R.lib()
    ext = C.CDLL(EXT, mode=C.RTLD_GLOBAL)
    ext.b200_duckdb_register.argtypes = [C.c_void_p]
    con = R.Connection(threads=4)
    assert ext.b200_duckdb_register(con.db) == 0
    with _Env({"B200_DISABLE": "1"}):
        con.execute(TABLE)
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
    """(pipe to a connection in a child process, has_device), as in test_gpu_duckdb_aggregate_types.py"""
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


# --------------------------------------------------------------------------------------- every function, filtered
def _functions(g):
    """count(*), count, sum, min, max, avg under filters (p is NULL in one row of 7; `g % 4 = 1` passes no row of
    three groups in four, nor of the NULL-key group), next to the same columns unfiltered"""
    return (f"count(*) FILTER (WHERE p) AS c_p, count(i32) FILTER (WHERE p) AS ci_p, "
            f"sum(i64) FILTER (WHERE g{g} % 4 = 1) AS s_g, min(i16) FILTER (WHERE p) AS min_i, "
            f"max(f64) FILTER (WHERE NOT p) AS max_f, avg(d92) FILTER (WHERE p) AS a_d, "
            f"sum(f64) FILTER (WHERE u8 > 100) AS s_f, avg(i32) FILTER (WHERE i16 > 0) AS a_i, "
            f"min(f64) FILTER (WHERE p) AS min_f, count(*) AS c, sum(i64) AS s")


FUNCTION_CASES = []
for _g in GROUP_COUNTS:
    for _t in [1, 4]:
        FUNCTION_CASES.append((f"functions-g{_g}-t{_t}", _t, _g, AGG_OPTIMIZERS, {}))
    FUNCTION_CASES.append((f"functions-g{_g}-t4-default", 4, _g, "", {}))
    if _g >= 200000:
        FUNCTION_CASES.append((f"functions-g{_g}-t1-nohc", 1, _g, AGG_OPTIMIZERS, {"B200_AGG_NO_HC": "1"}))


def _function_case(db, device, case):
    name, threads, g, optimizers, env = case
    sql = f"SELECT g{g}, {_functions(g)} FROM tf GROUP BY g{g} ORDER BY g{g}"
    exp, plan = _check(db, device, sql, _settings(threads, optimizers), env=env, by_value=FLOAT_MIN_MAX)
    assert len(exp[0].values) == g + 1, name
    s_g = exp[3]
    assert s_g.valid is not None and not s_g.valid.all() and s_g.valid.any(), name   # groups no row passes: NULL
    assert int(exp[10].values.sum()) == ROWS, name


@pytest.mark.parametrize("case", FUNCTION_CASES, ids=[c[0] for c in FUNCTION_CASES])
def test_filtered_aggregates_match_the_stock_operator(db, case):
    _function_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FUNCTION_CASES, ids=[c[0] for c in FUNCTION_CASES])
def test_filtered_aggregates_on_the_gpu_match_the_stock_operator(db, case):
    _function_case(db, True, case)


# ------------------------------------------------------------------------------------- PIVOT, limits, other shapes
_FILTERED12 = ", ".join([f"sum(i32) FILTER (WHERE pv = {v}) AS s{v}" for v in range(4)] +
                        [f"count(*) FILTER (WHERE pv = {v}) AS c{v}" for v in range(4)] +
                        ["min(i16) FILTER (WHERE p) AS mn", "max(i64) FILTER (WHERE p IS NULL) AS mx",
                         "sum(d92) FILTER (WHERE u8 < 7) AS sd", "count(f64) FILTER (WHERE NOT p) AS cf"])
_AGG13 = _FILTERED12 + ", count(*)"
# (name, query, decorated: True / False (the stock Hash Group By) / None (compared only) / the stock operator's name,
#  disabled optimizers, by_value columns)
SHAPES = [
    ("12-filtered-aggregates", f"SELECT g600, {_FILTERED12} FROM tf GROUP BY g600 ORDER BY g600", True,
     AGG_OPTIMIZERS, ()),
    ("13-aggregates-with-filters", f"SELECT g600, {_AGG13} FROM tf GROUP BY g600 ORDER BY g600", False,
     AGG_OPTIMIZERS, ()),
    ("pivot-in-list-sum-count", "SELECT * FROM (PIVOT tf ON pv IN (0, 1, 2, 3) USING sum(i32), count(*) "
                                "GROUP BY g600) ORDER BY g600", True, AGG_OPTIMIZERS, ()),
    ("pivot-sum-count", "SELECT * FROM (PIVOT tf ON pv USING sum(i64), count(*) GROUP BY g5) ORDER BY g5", True,
     AGG_OPTIMIZERS, ()),
    ("pivot-default-count", "SELECT * FROM (PIVOT tf ON pv GROUP BY g200000) ORDER BY g200000", True, "", ()),
    ("pivot-in-list-default-count", "SELECT * FROM (PIVOT tf ON pv IN (1, 3) GROUP BY g600, u8) ORDER BY g600, u8",
     True, AGG_OPTIMIZERS, ()),
    ("count-distinct-filter", "SELECT g600, count(DISTINCT u8) FILTER (WHERE p) AS cd FROM tf GROUP BY g600 "
                              "ORDER BY g600", None, AGG_OPTIMIZERS, ()),
    ("ungrouped-filter", "SELECT count(*) FILTER (WHERE p) AS c, sum(i64) FILTER (WHERE p) AS s, "
                         "min(f64) FILTER (WHERE p) AS min_f FROM tf", "Ungrouped Aggregate", AGG_OPTIMIZERS,
     FLOAT_MIN_MAX),
]
SHAPE_CASES = [(f"{s[0]}-t{t}", t) + s[1:] for s in SHAPES for t in [1, 4]]


def _check_stock(db, device, sql, settings, stock, by_value):
    """_check for a plan that must keep the stock operator named `stock` and no B200 operator"""
    pipe, has_device = db
    if device:
        assert has_device, "the gpu tests need a CUDA device"
    elif has_device:
        pytest.skip("with a CUDA device the decorator runs on it: the gpu-marked variant runs this case")
    pipe.send((settings, sql, {}, stock, "B200_", tuple(by_value)))
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(f"{result}\nquery: {sql}")
    plan, exp = result
    return exp, plan


def _shape_case(db, device, case):
    name, threads, sql, decorated, optimizers, by_value = case
    if isinstance(decorated, str):
        exp, plan = _check_stock(db, device, sql, _settings(threads, optimizers), decorated, by_value)
    else:
        exp, plan = _check(db, device, sql, _settings(threads, optimizers), decorated, by_value=by_value)
    assert len(exp[0].values) > 0, name
    if name.startswith("ungrouped") or name.startswith("13-"):
        assert "B200_" not in plan, plan


@pytest.mark.parametrize("case", SHAPE_CASES, ids=[c[0] for c in SHAPE_CASES])
def test_pivot_and_limits_match_the_stock_operator(db, case):
    _shape_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHAPE_CASES, ids=[c[0] for c in SHAPE_CASES])
def test_pivot_and_limits_on_the_gpu_match_the_stock_operator(db, case):
    _shape_case(db, True, case)
