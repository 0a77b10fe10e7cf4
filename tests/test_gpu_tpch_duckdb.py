"""The DuckDB operators of integration/ together: TPC-H's 22 queries, and synthetic chains in which one decorated
operator feeds another, through the decorated plans against the stock plans.

The harness is the one of tests/test_gpu_duckdb_operators.py: one connection in a spawned child process, every query
twice through the decorated plan and once with B200_DISABLE=1 (whose plan must name no B200_ operator), and the
results must agree in names, types, validity and values, floats bit for bit.  TPC-H holds money as DECIMAL, so every
SUM is exact and the DOUBLE results (AVG, DECIMAL division) are computed on the host from exact states: a float
difference is a wrong result, not a rounding to tolerate.

TPC-H defines the row order only up to ties on the ORDER BY keys, so rows that tie on them compare as a multiset.  For
a query with a LIMIT the stock plan runs once more without it: when a tie group crosses the cut, which rows of that
group the LIMIT keeps is not defined, and only their ORDER BY keys are compared (TIES_AT_THE_LIMIT names the queries
where this happens at SF 1).

With a CUDA device the tables are generated at SF 1: lineitem spans about 46 probe batches (B200_PROBE_BATCH =
131 072 rows), orders more than one build morsel (B200_MORSEL_ROWS = 1 048 576 rows), and Q18's GROUP BY l_orderkey
has 1.5 M groups.  PLANS pins the B200 operators each query's decorated plan contains at SF 1 under each
configuration, so no query can pass by being planned on the stock operators: the test fails when a recorded operator
disappears or falls back to "(host)".  Without a device every decorator forwards to the stock operator: the plumbing
variant runs the same queries at SF 0.01 and checks the results, and EXPLAINs SF 1 tables in a schema of their own to
check the joins and aggregates of PLANS, which do not depend on the device (AnalyseJoin / AnalyseAggregate), and that
every filter of PLANS is planned.

The synthetic chains (CHAINS) reach the paths between two decorated operators that TPC-H may miss or not reach at their
boundaries: a filter's slices as a join's build side over two morsels, a join's capacity-retried output probing a
second join, a join feeding an aggregate, an aggregate feeding a HAVING filter, and the mark column of a MARK join read
by a filter."""
import ctypes as C
import json
import os
import re

import pytest

from test_gpu_duckdb_operators import EXT, JOIN_OPTIMIZERS, MORSEL_ROWS, PROBE_BATCH, _assert_same, _Env

STOCK = {"B200_DISABLE": "1"}

# id -> (settings, environment at plan and run time)
CONFIGS = {
    "t4": ({"threads": 4}, {}),
    # one worker sees every chunk in order: the batch arithmetic is deterministic
    "t1": ({"threads": 1}, {}),
    # date and DECIMAL range predicates leave the scans and become B200_FILTERs
    "t4-scan": ({"threads": 4}, {"B200_SCAN_FILTERS": "1"}),
    # more GROUP BYs become hash aggregates, and every join table uses open addressing
    "t4-open": ({"threads": 4, "perfect_ht_threshold": 0}, {"B200_JOIN_NO_DENSE": "1"}),
}
QUERIES = range(1, 23)

# configuration -> query -> the B200 operators of the decorated plan at SF 1: (the join type of every B200_HASH_JOIN,
# sorted; B200_HASH_GROUP_BY count; batched B200_FILTER count; B200_FILTER(host) count).  Recorded on an H100 80GB
# HBM3.  The hash joins of TPC-H that stay on the stock operator carry a VARCHAR build payload, a second condition, an
# IS [NOT] DISTINCT FROM or expression key, or are RIGHT_SEMI / RIGHT_ANTI joins; the B200_FILTER(host)s hold string
# comparisons, IN lists, NOT or a CAST, which the kernel's program does not take.
PLANS = {
    "t4": {
        1: ("", 0, 0, 0),
        2: ("INNER", 1, 0, 0),
        3: ("INNER INNER", 1, 1, 0),
        4: ("", 0, 1, 0),
        5: ("INNER INNER", 0, 0, 0),
        6: ("", 0, 0, 0),
        7: ("", 0, 0, 2),
        8: ("INNER INNER INNER INNER INNER INNER", 0, 0, 0),
        9: ("INNER INNER", 0, 0, 0),
        10: ("INNER", 0, 0, 0),
        11: ("INNER INNER", 0, 0, 0),
        12: ("", 1, 0, 1),
        13: ("LEFT", 3, 0, 0),
        14: ("", 0, 0, 0),
        15: ("", 1, 0, 0),
        16: ("MARK MARK", 0, 1, 1),
        17: ("INNER SEMI", 2, 0, 0),
        18: ("", 1, 0, 1),
        19: ("", 0, 0, 2),
        20: ("INNER MARK SEMI", 2, 1, 0),
        21: ("INNER", 0, 2, 0),
        22: ("SEMI", 1, 2, 2),
    },
    "t1": {
        1: ("", 0, 0, 0),
        2: ("INNER", 1, 0, 0),
        3: ("INNER INNER", 1, 1, 0),
        4: ("", 0, 1, 0),
        5: ("INNER INNER", 0, 0, 0),
        6: ("", 0, 0, 0),
        7: ("", 0, 0, 2),
        8: ("INNER INNER INNER INNER INNER INNER", 0, 0, 0),
        9: ("INNER INNER", 0, 0, 0),
        10: ("INNER", 0, 0, 0),
        11: ("INNER INNER", 0, 0, 0),
        12: ("", 1, 0, 1),
        13: ("LEFT", 3, 0, 0),
        14: ("", 0, 0, 0),
        15: ("", 1, 0, 0),
        16: ("MARK MARK", 0, 1, 1),
        17: ("INNER SEMI", 2, 0, 0),
        18: ("", 1, 0, 1),
        19: ("", 0, 0, 2),
        20: ("INNER MARK SEMI", 2, 1, 0),
        21: ("INNER", 0, 2, 0),
        22: ("SEMI", 1, 2, 2),
    },
    "t4-scan": {
        1: ("", 0, 1, 0),
        2: ("INNER", 1, 1, 1),
        3: ("INNER INNER", 1, 3, 1),
        4: ("", 0, 2, 0),
        5: ("INNER INNER", 0, 2, 1),
        6: ("", 0, 1, 0),
        7: ("", 0, 2, 2),
        8: ("INNER INNER INNER INNER INNER INNER", 0, 2, 2),
        9: ("INNER INNER", 0, 0, 0),
        10: ("INNER", 0, 2, 1),
        11: ("INNER INNER", 0, 0, 1),
        12: ("", 1, 1, 1),
        13: ("LEFT", 3, 0, 0),
        14: ("", 0, 1, 0),
        15: ("", 1, 1, 0),
        16: ("MARK MARK", 0, 1, 2),
        17: ("INNER SEMI", 2, 1, 1),
        18: ("", 1, 1, 1),
        19: ("", 0, 0, 4),
        20: ("INNER MARK SEMI", 2, 2, 2),
        21: ("INNER", 0, 2, 2),
        22: ("SEMI", 1, 3, 2),
    },
    "t4-open": {
        1: ("", 1, 0, 0),
        2: ("INNER", 1, 0, 0),
        3: ("INNER INNER", 1, 1, 0),
        4: ("", 0, 1, 0),
        5: ("INNER INNER", 0, 0, 0),
        6: ("", 0, 0, 0),
        7: ("", 0, 0, 2),
        8: ("INNER INNER INNER INNER INNER INNER", 1, 0, 0),
        9: ("INNER INNER", 0, 0, 0),
        10: ("INNER", 0, 0, 0),
        11: ("INNER INNER", 0, 0, 0),
        12: ("", 1, 0, 1),
        13: ("LEFT", 3, 0, 0),
        14: ("", 0, 0, 0),
        15: ("", 1, 0, 0),
        16: ("MARK MARK", 0, 1, 1),
        17: ("INNER SEMI", 2, 0, 0),
        18: ("", 1, 0, 1),
        19: ("", 0, 0, 2),
        20: ("INNER MARK SEMI", 2, 1, 0),
        21: ("INNER", 0, 2, 0),
        22: ("SEMI", 1, 2, 2),
    },
}

# queries whose stock result at SF 1 has a tie group on the ORDER BY keys across the LIMIT: none (Q2, Q3, Q10 and Q21
# cut between distinct keys, Q18 has 57 rows)
TIES_AT_THE_LIMIT = set()


# ------------------------------------------------------------------------------------------------------ the plans
def _explain(con, sql, env):
    """the physical plan as a JSON tree"""
    with _Env(env):
        rows = con.fetchall("EXPLAIN (FORMAT json) " + sql)
    return json.loads(rows[0][-1])


def _operators(tree):
    """(name, join type or None) of every operator of the plan"""
    found = []

    def walk(node):
        if isinstance(node, list):
            for n in node:
                walk(n)
            return
        info = node.get("extra_info") or {}
        found.append((node.get("name", "").strip(), info.get("Join Type") if isinstance(info, dict) else None))
        walk(node.get("children", []))

    walk(tree)
    return found


def _b200_operators(ops, host):
    """the PLANS entry of a plan.  With `host` (no device) the joins and aggregates carry "(host)", and every filter is
    a B200_FILTER(host): the filters are returned as (0, their count)"""
    suffix = "(host)" if host else ""
    joins = " ".join(sorted(t or "?" for n, t in ops if n == "B200_HASH_JOIN" + suffix))
    aggs = sum(n == "B200_HASH_GROUP_BY" + suffix for n, _ in ops)
    return joins, aggs, sum(n == "B200_FILTER" for n, _ in ops), sum(n == "B200_FILTER(host)" for n, _ in ops)


# ------------------------------------------------------------------------------------------------- the comparison
def _order_keys(sql):
    """the result columns the outer ORDER BY names (TPC-H orders by bare output names)"""
    tail = re.split(r"(?i)\border\s+by\b", sql)
    if len(tail) == 1:
        return []
    tail = re.split(r"(?i)\blimit\b|;", tail[-1])[0]
    return [k.split()[0] for k in tail.split(",")]


def _cell(col, r):
    if col.valid is not None and not col.valid[r]:
        return (0,)
    v = col.values[r]
    if col.values.dtype.kind == "f":
        return (1, v.tobytes())
    return (1, v.item() if hasattr(v, "item") else v)


def _take(col, rows):
    from oracle import duckdb_ref as R

    valid = None if col.valid is None else col.valid[rows]
    return R.Column(col.name, col.values[rows], valid, col.type_id, col.scale)


def _assert_same_up_to_ties(got, exp, keys, what, keys_only_in_last_group=False):
    """`got` equals `exp` where rows that tie on the columns `keys` form a multiset; with `keys_only_in_last_group`
    only the keys of the last tie group are compared (a LIMIT cut through it)"""
    import numpy as np

    names = [c.name for c in exp]
    assert [c.name for c in got] == names, what
    kidx = [names.index(k) for k in keys]
    _assert_same([got[i] for i in kidx], [exp[i] for i in kidx], what + " (ORDER BY keys)")
    n = len(exp[0].values) if exp else 0
    starts = [r for r in range(n) if r == 0 or [_cell(exp[i], r) for i in kidx] != [_cell(exp[i], r - 1) for i in kidx]]
    if keys_only_in_last_group and starts:
        n = starts.pop()
    bounds = starts + [n]

    def canonical(cols):
        order = []
        for b, e in zip(bounds[:-1], bounds[1:]):
            order += sorted(range(b, e), key=lambda r: [_cell(c, r) for c in cols])
        order = np.array(order, dtype=np.int64)
        return [_take(c, order) for c in cols]

    _assert_same(canonical(got), canonical(exp), what)


def _settings(con, settings):
    con.execute("RESET perfect_ht_threshold")
    con.execute("RESET disabled_optimizers")
    for k, v in settings.items():
        con.execute(f"SET {k}='{v}'" if isinstance(v, str) else f"SET {k}={v}")


def _run_tpch(con, queries, config, nr):
    """in the child: the decorated plan's operators, two decorated runs against one stock run -> (PLANS entry, rows,
    whether a tie group crosses the LIMIT)"""
    settings, env = CONFIGS[config]
    _settings(con, settings)
    sql = queries[nr]
    ops = _b200_operators(_operators(_explain(con, sql, env)), host=False)
    with _Env(env):
        got = [con.execute(sql), con.execute(sql)]
    assert "B200_" not in json.dumps(_explain(con, sql, STOCK))
    with _Env(STOCK):
        exp = con.execute(sql)
    keys = _order_keys(sql)
    crossed = False
    limit = re.search(r"(?i)\blimit\s+(\d+)\s*;?\s*$", sql)
    if limit:
        with _Env(STOCK):
            full = con.execute(sql[:limit.start()])
        cut = int(limit.group(1))
        kidx = [[c.name for c in full].index(k) for k in keys]
        assert len(exp[0].values) == min(cut, len(full[0].values))
        crossed = len(full[0].values) > cut and \
            [_cell(full[i], cut - 1) for i in kidx] == [_cell(full[i], cut) for i in kidx]
    for i, g in enumerate(got):
        _assert_same_up_to_ties(g, exp, keys, f"Q{nr} {config} run {i + 1}", crossed)
    return ops, len(exp[0].values) if exp else 0, crossed


def _plan_sf1(con, queries, config, nr):
    """in the child without a device: the PLANS entry of the decorated plan over the SF 1 tables"""
    settings, env = CONFIGS[config]
    _settings(con, settings)
    con.execute("SET schema='sf1'")
    try:
        return _b200_operators(_operators(_explain(con, queries[nr], env)), host=True)
    finally:
        con.execute("SET schema='main'")


# ------------------------------------------------------------------------------------------------ synthetic chains
FB_ROWS = 3000000        # 1.8 M rows pass `lo < hi`: two build morsels on one worker
FB_FIRST_NULL = 1800000  # the first NULL key / payload: the 1 080 001st survivor, in the second morsel
CHAIN_PROBES = [PROBE_BATCH - 1, PROBE_BATCH + 1]
HAVING_ROWS = 1000000
assert FB_FIRST_NULL * 6 // 10 > MORSEL_ROWS and FB_ROWS * 6 // 10 < 2 * MORSEL_ROWS  # 6 rows in 10 pass the filter

CHAIN_TABLES = [
    # filter -> join build: `lo < hi` keeps the rows whose last digit is 0, 1, 2, 4, 5 or 7 - which the optimizer
    # cannot know, so the predicate stays in a LogicalFilter.  NULL keys and payloads only from FB_FIRST_NULL on (in
    # rows that pass); pa / pb are two INTEGER payloads, pc a BIGINT
    f"""CREATE TABLE fb AS SELECT (i % 10)::INTEGER AS lo, ((i * 7) % 10 + 1)::INTEGER AS hi,
           CASE WHEN i >= {FB_FIRST_NULL} AND i % 10 = 0 AND i % 7 = 0 THEN NULL ELSE i END AS bk,
           CASE WHEN i >= {FB_FIRST_NULL} AND i % 10 = 1 AND i % 3 = 0 THEN NULL ELSE (i * 3 - 5000000)::INTEGER END AS pa,
           CASE WHEN i >= {FB_FIRST_NULL} AND i % 10 = 2 AND i % 3 = 0 THEN NULL ELSE (7 - i)::INTEGER END AS pb,
           CASE WHEN i >= {FB_FIRST_NULL} AND i % 10 = 4 THEN NULL ELSE i * 1000000007 END AS pc
       FROM range({FB_ROWS}) r(i)""",
    # its probe side: every build row is hit about once in 8 probes of 400 000, NULL one row in 101
    f"""CREATE TABLE fp AS SELECT i AS pid, CASE WHEN i % 101 = 7 THEN NULL ELSE (i * 2654435761) % {FB_ROWS} END AS k
       FROM range(400000) r(i)""",
    # join -> join: jj1 holds every key 0 .. 39 999 five times (results of ~4x the probe: the capacity retry); its k2
    # payload probes jj2 (unique keys 0 .. 29 999 against k2 in 0 .. 49 999, NULL one row in 13)
    """CREATE TABLE jj1 AS SELECT i AS bid, (i % 40000)::INTEGER AS k,
           CASE WHEN i % 13 = 4 THEN NULL ELSE ((i * 7) % 50000)::INTEGER END AS k2,
           CASE WHEN i % 7 = 2 THEN NULL ELSE (i % 60000 - 30000)::SMALLINT END AS p2
       FROM range(200000) r(i)""",
    """CREATE TABLE jj2 AS SELECT i::INTEGER AS k, CASE WHEN i % 11 = 3 THEN NULL ELSE i * 1000003 END AS q8
       FROM range(30000) r(i)""",
    *[f"""CREATE TABLE jjp_{n} AS SELECT i AS pid,
            CASE WHEN i % 101 = 7 THEN NULL ELSE ((i * 2654435761) % 50000)::INTEGER END AS k
        FROM range({n}) r(i)""" for n in CHAIN_PROBES],
    # join -> aggregate: 250 000 unique build keys, every one hit by the 1.5 M probes; g5 / g200000 group on payloads
    """CREATE TABLE ja AS SELECT i::INTEGER AS k, CASE WHEN i % 1009 = 0 THEN NULL ELSE i % 5 END AS g5,
           CASE WHEN i % 1009 = 0 THEN NULL ELSE (i % 200000)::INTEGER END AS g200000,
           CASE WHEN i % 13 = 0 THEN NULL ELSE ((i * 7919) % 2000001 - 1000000)::INTEGER END AS v
       FROM range(250000) r(i)""",
    """CREATE TABLE jap AS SELECT i AS pid, ((i * 2654435761) % 250000)::INTEGER AS k FROM range(1500000) r(i)""",
    # aggregate -> filter: g200000 has 5 rows per group; b is NULL in every row of the groups g % 17 = 3
    f"""CREATE TABLE hv AS SELECT i % 5 AS g5, (i % 200000)::INTEGER AS g200000,
           ((i * 7919) % 1000003 - 500000)::INTEGER AS a,
           CASE WHEN i % 11 = 0 OR (i % 200000) % 17 = 3 THEN NULL ELSE ((i * 31337) % 1000003 - 500000)::INTEGER END AS b
       FROM range({HAVING_ROWS}) r(i)""",
    # MARK -> filter: k ~1/3 in 0 .. 299, NULL one row in 53; v > w in about half the rows, NULL in some
    *[f"""CREATE TABLE mf_{n} AS SELECT i AS pid,
            CASE WHEN i % 53 = 11 THEN NULL ELSE ((i * 2654435761) % 900)::INTEGER END AS k,
            CASE WHEN i % 29 = 4 THEN NULL ELSE ((i * 40503) % 1000)::INTEGER END AS v,
            ((i * 7919) % 1000)::INTEGER AS w
        FROM range({n}) r(i)""" for n in CHAIN_PROBES],
    "CREATE TABLE mfb AS SELECT (3 * i)::INTEGER AS k, CASE WHEN i = 17 THEN NULL ELSE (5 * i)::INTEGER END AS kn "
    "FROM range(100) r(i)",
]

FILTERED_BUILD = "(SELECT bk, pa, pb, pc FROM fb WHERE lo < hi)"


def _chains():
    """(name, threads, sql, the B200 operators the plan must contain, least result rows)"""
    join, agg, filt = "B200_HASH_JOIN", "B200_HASH_GROUP_BY", "B200_FILTER"
    cases = []
    # the INNER join's build side passes a second filter: `bk <= <largest probe key>`, from the probe side's statistics
    for kind, filters, rows in [("INNER", 2, 200000), ("LEFT", 1, 400000)]:
        for t in [1, 4]:
            cases.append((f"filter-build-{kind}-t{t}", t,
                          f"SELECT p.pid, b.bk, b.pa, b.pb, b.pc FROM fp p {kind} JOIN {FILTERED_BUILD} b ON p.k = b.bk "
                          "ORDER BY p.pid", {filt: filters, join: 1}, rows))
    for n in CHAIN_PROBES:
        first = f"jjp_{n} p JOIN jj1 b1 ON p.k = b1.k"
        cases.append((f"join-join-LEFT-{n}", 1,
                      f"SELECT p.pid, b1.bid, b1.p2, b1.k2, b2.q8 FROM {first} LEFT JOIN jj2 b2 ON b1.k2 = b2.k "
                      "ORDER BY p.pid, b1.bid", {join: 2}, 3 * n))
        cases.append((f"join-join-SEMI-{n}", 1,
                      f"SELECT p.pid, b1.bid, b1.p2 FROM {first} SEMI JOIN jj2 b2 ON b1.k2 = b2.k "
                      "ORDER BY p.pid, b1.bid", {join: 2}, n))
    for g in [5, 200000]:
        for t in [1, 4]:
            cases.append((f"join-aggregate-g{g}-t{t}", t,
                          f"SELECT b.g{g}, count(*), count(b.v), sum(b.v), min(b.v), max(b.v) "
                          f"FROM jap p JOIN ja b ON p.k = b.k GROUP BY b.g{g} ORDER BY b.g{g}",
                          {join: 1, agg: 1}, g * 99 // 100))
    for g in [5, 200000]:
        for t in [1, 4]:
            cases.append((f"having-min-max-g{g}-t{t}", t,
                          f"SELECT g{g}, min(a), max(b), count(*) FROM hv GROUP BY g{g} HAVING min(a) < max(b) "
                          f"ORDER BY g{g}", {agg: 1, filt: 1}, 1 if g == 5 else g // 4))
            cases.append((f"having-counts-g{g}-t{t}", t,
                          f"SELECT g{g}, count(*), count(b) FROM hv GROUP BY g{g} HAVING count(*) > count(b) "
                          f"ORDER BY g{g}", {agg: 1, filt: 1}, 1 if g == 5 else g // 20))
    for n in CHAIN_PROBES:
        cases.append((f"mark-filter-{n}", 1, f"SELECT pid, k, v, w FROM mf_{n} WHERE k IN (SELECT k FROM mfb) OR v > w "
                                             "ORDER BY pid", {join: 1, filt: 1}, n // 3))
        cases.append((f"mark-filter-null-build-{n}", 1,
                      f"SELECT pid, k, v, w FROM mf_{n} WHERE k IN (SELECT kn FROM mfb) OR v > w ORDER BY pid",
                      {join: 1, filt: 1}, n // 3))
    cases.append(("mark-filter-t4", 4, f"SELECT pid, k, v, w FROM mf_{CHAIN_PROBES[1]} WHERE k IN (SELECT kn FROM mfb) "
                                       "OR v > w ORDER BY pid", {join: 1, filt: 1}, CHAIN_PROBES[1] // 3))
    return cases


CHAINS = _chains()


def _run_chain(con, name, threads, sql, operators, least_rows, has_device):
    """in the child: every operator of the chain planned (on the device with one), two decorated runs against one stock
    run, in the order of the unique ORDER BY key"""
    # keep the sides as written (the right side is the build side), no projection that narrows the join keys between
    # two operators of the chain, and every GROUP BY a hash aggregate
    _settings(con, {"threads": threads, "disabled_optimizers": JOIN_OPTIMIZERS + ",compressed_materialization",
                    "perfect_ht_threshold": 0})
    ops = _operators(_explain(con, sql, {}))
    names = [n for n, _ in ops]
    for op, count in operators.items():
        want = op if has_device else op + "(host)"
        assert names.count(want) == count, (name, want, ops)
        if has_device:
            assert op + "(host)" not in names, (name, ops)
    if name.startswith("mark"):
        assert any(t == "MARK" for n, t in ops if n.startswith("B200_HASH_JOIN")), (name, ops)
    with _Env({}):
        got = [con.execute(sql), con.execute(sql)]
    assert "B200_" not in json.dumps(_explain(con, sql, STOCK))
    with _Env(STOCK):
        exp = con.execute(sql)
    rows = len(exp[0].values)
    assert rows >= least_rows, (name, rows, least_rows)
    for i, g in enumerate(got):
        _assert_same(g, exp, f"{name} run {i + 1}: {sql}")
    return rows


# ---------------------------------------------------------------------------------------------------- the child
def _serve(pipe):
    """the child process of db(): owns the connection and answers requests until it receives None"""
    from oracle import duckdb_ref as R

    R.lib()  # the reference library first, so the binding resolves its DuckDB symbols against the same copy
    ext = C.CDLL(EXT, mode=C.RTLD_GLOBAL)
    ext.b200_duckdb_register.argtypes = [C.c_void_p]
    con = R.Connection(threads=4)
    assert ext.b200_duckdb_register(con.db) == 0
    has_device = ext.b200_device_count() > 0
    with _Env(STOCK):
        con.execute(f"CALL dbgen(sf={1 if has_device else 0.01})")
        if not has_device:
            con.execute("CREATE SCHEMA sf1")
            con.execute("CALL dbgen(sf=1, schema='sf1')")
        for sql in CHAIN_TABLES:
            con.execute(sql)
        queries = dict(con.fetchall("SELECT query_nr, query FROM tpch_queries()"))
    pipe.send(has_device)
    handlers = {
        "tpch": lambda config, nr: _run_tpch(con, queries, config, nr),
        "plan": lambda config, nr: _plan_sf1(con, queries, config, nr),
        "chain": lambda *case: _run_chain(con, *case, has_device),
    }
    while True:
        request = pipe.recv()
        if request is None:
            break
        try:
            pipe.send(("ok", handlers[request[0]](*request[1:])))
        except Exception as e:  # a failed assertion or query fails the test that sent it
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


def _ask(db, device, *request):
    pipe, has_device = db
    if device:
        assert has_device, "the gpu tests need a CUDA device"
    elif has_device:
        pytest.skip("with a CUDA device the decorators run on it: the gpu-marked variant runs this case")
    pipe.send(request)
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(f"{result}\nrequest: {request[:3]}")
    return result


# ------------------------------------------------------------------------------------------------------- TPC-H
TPCH_CASES = [(config, nr) for config in CONFIGS for nr in QUERIES]
TPCH_IDS = [f"{config}-q{nr:02d}" for config, nr in TPCH_CASES]


@pytest.mark.parametrize("case", TPCH_CASES, ids=TPCH_IDS)
def test_tpch_sf001_matches_the_stock_plan(db, case):
    _ask(db, False, "tpch", *case)


@pytest.mark.parametrize("case", TPCH_CASES, ids=TPCH_IDS)
def test_tpch_sf1_plans_decorate_the_pinned_joins_and_aggregates(db, case):
    config, nr = case
    joins, aggs, _, filters = _ask(db, False, "plan", config, nr)
    pinned = PLANS[config][nr]
    assert (joins, aggs, filters) == (pinned[0], pinned[1], pinned[2] + pinned[3]), (case, pinned)


@pytest.mark.gpu
@pytest.mark.parametrize("case", TPCH_CASES, ids=TPCH_IDS)
def test_tpch_sf1_on_the_gpu_matches_the_stock_plan(db, case):
    config, nr = case
    ops, rows, crossed = _ask(db, True, "tpch", config, nr)
    assert ops == PLANS[config][nr], (case, "the decorated operators differ from the pinned plan", ops, PLANS[config][nr])
    assert rows > 0, case
    assert crossed == (nr in TIES_AT_THE_LIMIT), (case, "a tie group crosses the LIMIT" if crossed else "")


# ------------------------------------------------------------------------------------------------------ chains
@pytest.mark.parametrize("case", CHAINS, ids=[c[0] for c in CHAINS])
def test_chained_operators_match_the_stock_plan(db, case):
    _ask(db, False, "chain", *case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAINS, ids=[c[0] for c in CHAINS])
def test_chained_operators_on_the_gpu_match_the_stock_plan(db, case):
    _ask(db, True, "chain", *case)
