"""RIGHT and FULL OUTER hash joins through B200HashJoin against the stock operator, in the way of
tests/test_gpu_duckdb_operators.py: every query runs in one connection twice through the decorated plan and once with
B200_DISABLE=1, and the results must agree bit for bit.  The EXPLAIN of the decorated plan must show B200_HASH_JOIN
over a RIGHT or FULL join - without "(host)" on a GPU.  The unmatched build rows come from the operator's source phase,
after every probe: NULL probe-side columns (VARCHAR included) and the build columns.

Probe sizes sit at the 128 K-row batch boundary (B200_PROBE_BATCH) with threads=1; the 2.5 M-row build side spans
several build morsels and several 1 Mi-row scan ranges, at threads 1 and 4.  With the optimizer on, a small LEFT JOIN
big query reaches the decorator as a RIGHT join (DuckDB builds on the smaller side and flips the join type).  Joins
the decorator does not take - RIGHT_SEMI, RIGHT_ANTI, a VARCHAR build payload, a residual predicate - keep the stock
operator.  Without a CUDA device the decorator forwards to the stock operator and the plumbing variants check the
"(host)" plan and the same results."""
import ctypes as C
import os

import pytest

from test_gpu_duckdb_operators import EXT, JOIN_OPTIMIZERS, PROBE_BATCH, TABLES as OP_TABLES, _compare, _Env, _plan, \
    _probe_table

PROBE_SIZES = [PROBE_BATCH - 1, PROBE_BATCH, PROBE_BATCH + 1, 1000003]
# jb (100 000 rows, unique even keys with NULLs, payloads with NULLs), jb5 (duplicate keys), jbig (2.5 M rows)
TABLES = OP_TABLES[:3] + [_probe_table(n) for n in PROBE_SIZES] + [
    "CREATE TABLE jbv AS SELECT i AS bid, (2 * i)::INTEGER AS ki, 'build-' || i AS sv FROM range(50000) r(i)",
]
PAYLOAD = ("bid", "p1", "p2", "p4", "p8", "pd")
EMPTY_BUILD = "(SELECT * FROM jb WHERE bid % 2 = 2)"


def _sql(kind, probe, build, key, build_key=None, payload=PAYLOAD, probe_cols=("pid",)):
    lhs = ", ".join("p." + c for c in probe_cols)
    rhs = ", ".join("b." + c for c in payload)
    return (f"SELECT {lhs}, {rhs} FROM {probe} p {kind} JOIN {build} b ON p.{key} = b.{build_key or key} "
            f"ORDER BY p.pid, b.bid")


def _cases():
    cases = []
    for kind in ["RIGHT", "FULL"]:
        for n in PROBE_SIZES[:3]:
            cases.append((f"batch-{n}-{kind}-t1", 1, _sql(kind, f"jp_{n}", "jb", "ki")))
        cases.append((f"batch-1000003-{kind}-t4", 4, _sql(kind, "jp_1000003", "jb", "ki")))
        for key in ["kb", "kd", "ks"]:             # key types; ks repeats: duplicate build keys
            cases.append((f"key-{key}-{kind}", 1, _sql(kind, "jp_131073", "jb", key)))
        cases.append((f"duplicates-{kind}", 1, _sql(kind, "jp_131073", "jb5", "kh", "k", ("bid", "p2"))))
        cases.append((f"varchar-probe-{kind}", 1, _sql(kind, "jp_131073", "jb", "ki", probe_cols=("pid", "s"))))
        cases.append((f"build-key-out-{kind}", 1, _sql(kind, "jp_131073", "jb", "ki", payload=("bid", "ki", "p4"))))
        for t in [1, 4]:                            # several build morsels and scan ranges
            cases.append((f"build-morsels-{kind}-t{t}", t,
                          _sql(kind, "jp_1000003", "jbig", "kg", "k", ("bid", "p8"))))
        cases.append((f"empty-build-{kind}", 1, _sql(kind, "jp_131073", EMPTY_BUILD, "ki")))
        cases.append((f"empty-probe-{kind}", 1, _sql(kind, "(SELECT * FROM jp_131073 WHERE pid % 2 = 2)", "jb", "ki")))
    return cases


CASES = _cases()
# with the optimizer on: (name, sql, what the decorated plan must show)
OPTIMIZED = [
    ("small-left-join-big", "SELECT b.bid, b.p4, p.pid, p.s FROM jb b LEFT JOIN jp_1000003 p ON b.ki = p.ki "
                            "ORDER BY b.bid, p.pid", "RIGHT"),
    ("full-join-group-by", "SELECT b.p1, count(*), count(p.pid), sum(b.p8), min(p.pid) FROM jp_131073 p "
                           "FULL JOIN jb b ON p.ki = b.ki GROUP BY b.p1 ORDER BY b.p1", "B200_HASH_GROUP_BY"),
]
# joins the decorator leaves to the stock operator: (name, settings, sql, join type the stock plan shows)
STOCK = [
    ("right-semi", "", "SELECT b.bid FROM jb b SEMI JOIN jp_1000003 p ON b.ki = p.ki ORDER BY b.bid", "RIGHT_SEMI"),
    ("right-anti", "", "SELECT b.bid FROM jb b ANTI JOIN jp_1000003 p ON b.ki = p.ki ORDER BY b.bid", "RIGHT_ANTI"),
    ("right-varchar-payload", JOIN_OPTIMIZERS,
     "SELECT p.pid, b.bid, b.sv FROM jp_131073 p RIGHT JOIN jbv b ON p.ki = b.ki ORDER BY p.pid, b.bid", "RIGHT"),
    ("full-residual", JOIN_OPTIMIZERS,
     "SELECT p.pid, b.bid FROM jp_131073 p FULL JOIN jb b ON p.ki = b.ki AND p.pid < b.bid * 3 "
     "ORDER BY p.pid, b.bid", "FULL"),
]


def _serve(pipe):
    """the child process of db(): owns the connection and runs _compare / plan requests until it receives None"""
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
            if request[0] == "plan":
                settings, sql = request[1:]
                for k, v in settings.items():
                    con.execute(f"SET {k}='{v}'" if isinstance(v, str) else f"SET {k}={v}")
                pipe.send(("ok", (_plan(con, sql, {}), con.execute(sql))))
            else:
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


def _request(db, device, request):
    pipe, has_device = db
    if device:
        assert has_device, "the gpu tests need a CUDA device"
    elif has_device:
        pytest.skip("with a CUDA device the decorator runs on it: the gpu-marked variant runs this case")
    pipe.send(request)
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(f"{result}\nquery: {request}")
    return result


def _planned(device):
    return ("B200_HASH_JOIN", "B200_HASH_JOIN(host)") if device else ("B200_HASH_JOIN(host)", None)


def _outer_case(db, device, case):
    name, threads, sql = case
    settings = {"threads": threads, "disabled_optimizers": JOIN_OPTIMIZERS, "perfect_ht_threshold": 0}
    planned, not_planned = _planned(device)
    plan, exp = _request(db, device, (settings, sql, {}, planned, not_planned))
    assert ("RIGHT" if "RIGHT" in name else "FULL") in plan, plan
    rows = len(exp[0].values)
    nulls_left = 0 if exp[0].valid is None else int((~exp[0].valid).sum())
    if name.startswith("empty-build"):
        assert rows == (0 if "RIGHT" in name else 131073), (name, rows)
    elif name.startswith("empty-probe"):
        assert rows == 100000 and nulls_left == rows, (name, rows)   # every build row, from the scan
    else:
        assert 0 < nulls_left < rows, (name, nulls_left, rows)      # the probe and the scan both emitted rows


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_outer_join_matches_the_stock_operator(db, case):
    _outer_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_outer_join_on_the_gpu_matches_the_stock_operator(db, case):
    _outer_case(db, True, case)


def _optimized_case(db, device, case):
    name, sql, shows = case
    settings = {"threads": 4, "disabled_optimizers": "", "perfect_ht_threshold": 0}
    planned, not_planned = _planned(device)
    plan, exp = _request(db, device, (settings, sql, {}, planned, not_planned))
    assert shows in plan, plan
    if name == "small-left-join-big":
        assert "LEFT" not in plan.replace("LEFT_", ""), plan     # the decorated join is the flipped RIGHT join
        assert len(exp[0].values) > 100000


@pytest.mark.parametrize("case", OPTIMIZED, ids=[c[0] for c in OPTIMIZED])
def test_optimized_plans_match_the_stock_operator(db, case):
    _optimized_case(db, False, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", OPTIMIZED, ids=[c[0] for c in OPTIMIZED])
def test_optimized_plans_on_the_gpu_match_the_stock_operator(db, case):
    _optimized_case(db, True, case)


@pytest.mark.parametrize("case", STOCK, ids=[c[0] for c in STOCK])
def test_other_joins_stay_stock(db, case):
    """the plan holds the join type named and no B200_ operator, with or without a device"""
    name, optimizers, sql, join_type = case
    pipe, _ = db
    pipe.send(("plan", {"threads": 4, "disabled_optimizers": optimizers, "perfect_ht_threshold": 0}, sql))
    status, result = pipe.recv()
    assert status == "ok", result
    plan, _ = result
    assert join_type in plan and "B200_" not in plan, plan
