#!/usr/bin/env python3
"""Generate the golden fixtures in this directory by running the UNMODIFIED reference
(oracle/_ref/libduckdb_ref.so, built by oracle/build_ref.py from the reference's sources).

    python tests/golden/make_golden.py

Outputs (committed):
  hash_kat.npz     inputs of every supported type (+ NULLs, multi-column) and DuckDB's hash() of them
  tpch_sf001.npz   TPC-H SF0.01 (CALL dbgen(sf=0.01)) columns used by the BASELINE configs and the
                   reference's answers: config 1 (filter scan), Q1 (hash aggregate, perfect_ht_threshold=0),
                   Q14 join (lineitem x part), Q3-shaped join + group-by
  filter_cases.npz random columns + the reference's result for a set of predicates (NULLs, NaN, AND/OR)
  join_cases.npz   random key columns with duplicates/NULLs and the reference's inner/left/semi/anti/mark results
  reference_results.json  the reference's answers for the tests that compare with it (see reference_results())
  reference_avg.npz       the reference's avg(d) of every group of test_gpu_parity's group-by, as the exact bit
                          difference from numpy's bincount mean (mostly 0 to a few units in the last place: the file stays small)
  expr_cases.json  the reference's result (or "error") of numeric CASTs and checked integer + - * at the edges
                   (expr_edge_cases())
  join_edge_cases.npz  composite-key joins with NULLs, +-0.0, NaN and type limits, and single-key MARK joins against
                   all-NULL, empty and NULL-holding build sides
"""
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import bincount_mean, digest, digest_array, py_scalar  # noqa: E402
from oracle import duckdb_ref as R  # noqa: E402
from oracle.build_ref import REF  # noqa: E402  (DUCKDB_REF: the reference's source tree)

OUT = os.path.dirname(os.path.abspath(__file__))
rng = np.random.default_rng(42)


def col_arrays(c):
    return c.values, (np.ones(len(c.values), dtype=bool) if c.valid is None else c.valid)


def hash_kat(con):
    out = {}
    n = 257
    specs = {
        "i8": np.int8, "i16": np.int16, "i32": np.int32, "i64": np.int64,
        "u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64,
    }
    for name, dt in specs.items():
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, size=n, dtype=dt, endpoint=True)
        v[:4] = [0, 1, info.max, info.min]
        valid = rng.random(n) > 0.2
        con.load_table(f"t_{name}", {"v": (v, valid)})
        h = con.execute(f"SELECT hash(v) FROM t_{name}")[0].values
        out[f"{name}_v"], out[f"{name}_valid"], out[f"{name}_h"] = v, valid, h
    for name, dt in {"f32": np.float32, "f64": np.float64}.items():
        v = rng.standard_normal(n).astype(dt)
        v[:6] = [0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf]
        valid = rng.random(n) > 0.2
        valid[:6] = True
        con.load_table(f"t_{name}", {"v": (v, valid)})
        h = con.execute(f"SELECT hash(v) FROM t_{name}")[0].values
        out[f"{name}_v"], out[f"{name}_valid"], out[f"{name}_h"] = v, valid, h
    b = rng.random(n) > 0.5
    con.load_table("t_b", {"v": b})
    out["bool_v"], out["bool_h"] = b, con.execute("SELECT hash(v) FROM t_b")[0].values
    # multi-column combine: hash(a, b, c)
    a = rng.integers(-5, 5, size=n).astype(np.int64)
    bb = rng.integers(0, 3, size=n).astype(np.uint16)
    c = rng.integers(-2, 2, size=n).astype(np.int8)
    av, bv = rng.random(n) > 0.1, rng.random(n) > 0.1
    con.load_table("t_multi", {"a": (a, av), "b": (bb, bv), "c": c})
    out["multi_a"], out["multi_a_valid"], out["multi_b"], out["multi_b_valid"], out["multi_c"] = a, av, bb, bv, c
    out["multi_h"] = con.execute("SELECT hash(a, b, c) FROM t_multi")[0].values
    np.savez_compressed(os.path.join(OUT, "hash_kat.npz"), **out)


def tpch(con):
    con.execute("CALL dbgen(sf=0.01)")
    out = {}
    li = con.execute("SELECT l_orderkey, l_partkey, l_quantity, l_extendedprice, l_discount, l_tax, "
                     "l_returnflag, l_linestatus, l_shipdate FROM lineitem")
    names = ["l_orderkey", "l_partkey", "l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag",
             "l_linestatus", "l_shipdate"]
    for nme, c in zip(names, li):
        if c.values.dtype == object:  # flags: single characters -> uint8 codes
            out[nme] = np.array([ord(x) for x in c.values], dtype=np.uint8)
        else:
            out[nme] = c.values
    # config 1
    r = con.execute("SELECT l_quantity FROM lineitem WHERE l_shipdate < DATE '1994-01-01'")
    out["cfg1_quantity"] = r[0].values
    out["cfg1_date_const"] = np.array(con.execute("SELECT DATE '1994-01-01'")[0].values)
    # Q1 through the named operator (HASH_GROUP_BY)
    con.execute("SET perfect_ht_threshold=0")
    q1 = con.execute(
        "SELECT l_returnflag, l_linestatus, sum(l_quantity), sum(l_extendedprice), "
        "sum(l_extendedprice*(1-l_discount)), sum(l_extendedprice*(1-l_discount)*(1+l_tax)), "
        "avg(l_quantity), avg(l_extendedprice), avg(l_discount), count(*) "
        "FROM lineitem WHERE l_shipdate <= DATE '1998-12-01' - INTERVAL '90' DAY "
        "GROUP BY l_returnflag, l_linestatus ORDER BY 1, 2")
    out["q1_date_const"] = np.array(con.execute("SELECT (DATE '1998-12-01' - INTERVAL '90' DAY)::DATE")[0].values)
    out["q1_returnflag"] = np.array([ord(x) for x in q1[0].values], dtype=np.uint8)
    out["q1_linestatus"] = np.array([ord(x) for x in q1[1].values], dtype=np.uint8)
    for i, nme in enumerate(["sum_qty", "sum_base_price", "sum_disc_price", "sum_charge"]):
        out["q1_" + nme] = np.array([int(x) for x in q1[2 + i].values], dtype=object).astype(np.float64)
        out["q1_" + nme + "_str"] = np.array([str(int(x)) for x in q1[2 + i].values])
    for i, nme in enumerate(["avg_qty", "avg_price", "avg_disc"]):
        out["q1_" + nme] = q1[6 + i].values
    out["q1_count"] = q1[9].values
    # Q14 join: part build side, promo flag payload
    p = con.execute("SELECT p_partkey, (p_type LIKE 'PROMO%')::UTINYINT FROM part")
    out["p_partkey"], out["p_promo"] = p[0].values, p[1].values
    j = con.execute(
        "SELECT l_orderkey, l_partkey, l_extendedprice, l_discount, (p_type LIKE 'PROMO%')::UTINYINT AS promo "
        "FROM lineitem, part WHERE l_partkey = p_partkey AND l_shipdate >= DATE '1995-09-01' "
        "AND l_shipdate < DATE '1995-10-01' ORDER BY l_orderkey, l_partkey, l_extendedprice")
    out["q14_lo"], out["q14_hi"] = (np.array(con.execute("SELECT DATE '1995-09-01'")[0].values),
                                    np.array(con.execute("SELECT DATE '1995-10-01'")[0].values))
    for nme, c in zip(["q14_orderkey", "q14_partkey", "q14_price", "q14_discount", "q14_promo"], j):
        out[nme] = c.values
    out["q14_result"] = con.execute(
        "SELECT 100.00 * sum(CASE WHEN p_type LIKE 'PROMO%' THEN l_extendedprice*(1-l_discount) ELSE 0 END) / "
        "sum(l_extendedprice*(1-l_discount)) FROM lineitem, part WHERE l_partkey = p_partkey AND "
        "l_shipdate >= DATE '1995-09-01' AND l_shipdate < DATE '1995-10-01'")[0].values
    # Q3-shaped: orders x lineitem join + 3-key group-by
    o = con.execute("SELECT o_orderkey, o_orderdate, o_shippriority FROM orders")
    out["o_orderkey"], out["o_orderdate"], out["o_shippriority"] = o[0].values, o[1].values, o[2].values
    q3 = con.execute(
        "SELECT l_orderkey, o_orderdate, o_shippriority, sum(l_extendedprice*(1-l_discount)) AS revenue, count(*) "
        "FROM orders, lineitem WHERE l_orderkey = o_orderkey AND o_orderdate < DATE '1995-03-15' "
        "AND l_shipdate > DATE '1995-03-15' GROUP BY l_orderkey, o_orderdate, o_shippriority ORDER BY 1, 2, 3")
    out["q3_date"] = np.array(con.execute("SELECT DATE '1995-03-15'")[0].values)
    out["q3_orderkey"], out["q3_orderdate"], out["q3_shippriority"] = q3[0].values, q3[1].values, q3[2].values
    out["q3_revenue_str"] = np.array([str(int(x)) for x in q3[3].values])
    out["q3_count"] = q3[4].values
    con.execute("RESET perfect_ht_threshold")
    np.savez_compressed(os.path.join(OUT, "tpch_sf001.npz"), **out)


def filter_cases(con):
    n = 5000
    out = {}
    a = rng.integers(-50, 50, size=n).astype(np.int32)
    av = rng.random(n) > 0.15
    b = rng.integers(-50, 50, size=n).astype(np.int32)
    bv = rng.random(n) > 0.15
    d = rng.standard_normal(n)
    d[rng.random(n) < 0.05] = np.nan
    d[rng.random(n) < 0.05] = 0.0
    d[rng.random(n) < 0.02] = -0.0
    dv = rng.random(n) > 0.1
    e = rng.integers(0, 1 << 62, size=n).astype(np.int64)
    con.load_table("f", {"a": (a, av), "b": (b, bv), "d": (d, dv), "e": e})
    out.update(a=a, a_valid=av, b=b, b_valid=bv, d=d, d_valid=dv, e=e)
    preds = {
        "lt_const": "a < 7", "eq_cols": "a = b", "ne_cols": "a <> b", "ge_cols": "a >= b",
        "and2": "a < 10 AND b > -10", "or2": "a < -20 OR b > 20", "and_or": "(a < 0 AND b > 0) OR a = b",
        "isnull": "a IS NULL", "isnotnull_and": "a IS NOT NULL AND b < 3",
        "distinct": "a IS DISTINCT FROM b", "notdistinct": "a IS NOT DISTINCT FROM b",
        "dbl_gt": "d > 0.5", "dbl_nan_eq": "d = 'NaN'::DOUBLE", "dbl_ge_nan": "d >= 'NaN'::DOUBLE",
        "dbl_lt_nan": "d < 'NaN'::DOUBLE", "dbl_eq_zero": "d = 0.0", "not_lt": "NOT (a < b)",
        "big": "e > 2305843009213693952",
    }
    for name, p in preds.items():
        r = con.execute(f"SELECT rowid FROM f WHERE {p} ORDER BY rowid")[0].values
        out["sel_" + name] = r.astype(np.uint32)
    # projection with arithmetic: a + b (INTEGER), e * 2 (BIGINT)
    r = con.execute("SELECT a + b, rowid FROM f WHERE a < 7 ORDER BY rowid")
    out["proj_add"], out["proj_add_valid"] = col_arrays(r[0])
    np.savez_compressed(os.path.join(OUT, "filter_cases.npz"), **out)


def join_cases(con):
    out = {}
    nb, npb = 700, 3000
    bk = rng.integers(0, 400, size=nb).astype(np.int64)
    bkv = rng.random(nb) > 0.05
    bp = rng.integers(-1000, 1000, size=nb).astype(np.int32)
    pk = rng.integers(0, 500, size=npb).astype(np.int64)
    pkv = rng.random(npb) > 0.05
    con.load_table("jb", {"k": (bk, bkv), "p": bp})
    con.load_table("jp", {"k": (pk, pkv), "id": np.arange(npb, dtype=np.int32)})
    out.update(bk=bk, bk_valid=bkv, bp=bp, pk=pk, pk_valid=pkv)
    con.execute("SET disabled_optimizers='join_filter_pushdown'")
    r = con.execute("SELECT jp.id, jb.p FROM jp JOIN jb ON jp.k = jb.k ORDER BY 1, 2")
    out["inner_id"], out["inner_p"] = r[0].values, r[1].values
    r = con.execute("SELECT jp.id, jb.p FROM jp LEFT JOIN jb ON jp.k = jb.k ORDER BY 1, 2")
    out["left_id"] = r[0].values
    out["left_p"], out["left_p_valid"] = col_arrays(r[1])
    out["semi_id"] = con.execute("SELECT id FROM jp SEMI JOIN jb ON jp.k = jb.k ORDER BY 1")[0].values
    out["anti_id"] = con.execute("SELECT id FROM jp ANTI JOIN jb ON jp.k = jb.k ORDER BY 1")[0].values
    r = con.execute("SELECT id, k IN (SELECT k FROM jb) FROM jp ORDER BY 1")
    out["mark"], out["mark_valid"] = col_arrays(r[1])
    # composite key (2 columns) inner join count + checksum
    b2 = rng.integers(0, 20, size=nb).astype(np.int16)
    p2 = rng.integers(0, 20, size=npb).astype(np.int16)
    con.load_table("jb2", {"k": (bk, bkv), "k2": b2, "p": bp})
    con.load_table("jp2", {"k": (pk, pkv), "k2": p2, "id": np.arange(npb, dtype=np.int32)})
    r = con.execute("SELECT jp2.id, jb2.p FROM jp2 JOIN jb2 ON jp2.k = jb2.k AND jp2.k2 = jb2.k2 ORDER BY 1, 2")
    out.update(b2=b2, p2=p2)
    out["inner2_id"], out["inner2_p"] = r[0].values, r[1].values
    np.savez_compressed(os.path.join(OUT, "join_cases.npz"), **out)


def join_edge_keys(rng, n):
    """composite join keys (BIGINT, DOUBLE, SMALLINT) drawn from small pools of edge values (type limits, +-0.0, NaN,
    infinities) so that duplicates and cross-side matches are common, with NULLs in every key position"""
    a = rng.choice(np.array([-2 ** 63, 2 ** 63 - 1, 0, 1, -1, 2 ** 62], dtype=np.int64), size=n)
    d = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -np.inf, np.inf, np.finfo(np.float64).max], dtype=np.float64),
                   size=n)
    s = rng.choice(np.array([-32768, 32767, 0, -1], dtype=np.int16), size=n)
    valid = [rng.random(n) > 0.08 for _ in range(3)]
    return (a, valid[0]), (d, valid[1]), (s, valid[2])


def join_edge_cases(con):
    """join_edge_cases.npz: the semantics the oracle is pinned on beyond join_cases.npz.
    Composite keys (BIGINT, DOUBLE, SMALLINT) with NULLs in every position, +-0.0, NaN and the type limits: INNER,
    LEFT, SEMI and ANTI results as (probe id, build id) pairs.  Single-key MARK (`k IN (SELECT k FROM b)`) against a
    build side of only NULL keys, an empty one and one with a NULL key among others."""
    rng = np.random.default_rng(2024)   # its own generator: the file regenerates identically when run by name
    out = {}
    nb, npb = 300, 400
    bcols, pcols = join_edge_keys(rng, nb), join_edge_keys(rng, npb)
    con.load_table("cb", {"a": bcols[0], "d": bcols[1], "s": bcols[2], "id": np.arange(nb, dtype=np.int32)})
    con.load_table("cp", {"a": pcols[0], "d": pcols[1], "s": pcols[2], "id": np.arange(npb, dtype=np.int32)})
    for side, cols in (("b", bcols), ("p", pcols)):
        for name, (v, valid) in zip("ads", cols):
            out[f"{side}_{name}"], out[f"{side}_{name}_valid"] = v, valid
    con.execute("SET disabled_optimizers='join_filter_pushdown'")
    on = "cp.a = cb.a AND cp.d = cb.d AND cp.s = cb.s"
    r = con.fetchall(f"SELECT cp.id, cb.id FROM cp JOIN cb ON {on} ORDER BY 1, 2")
    out["inner"] = np.array(r, dtype=np.int32).reshape(-1, 2)
    r = con.fetchall(f"SELECT cp.id, cb.id FROM cp LEFT JOIN cb ON {on}")
    out["left"] = np.array(sorted((p, -1 if b is None else b) for p, b in r), dtype=np.int32).reshape(-1, 2)
    out["semi"] = con.execute(f"SELECT id FROM cp SEMI JOIN cb ON {on} ORDER BY 1")[0].values.astype(np.int32)
    out["anti"] = con.execute(f"SELECT id FROM cp ANTI JOIN cb ON {on} ORDER BY 1")[0].values.astype(np.int32)
    # single-key MARK
    npm = 50
    mk = rng.integers(0, 8, size=npm).astype(np.int64)
    mkv = rng.random(npm) > 0.2
    con.load_table("mp", {"k": (mk, mkv), "id": np.arange(npm, dtype=np.int32)})
    out["mp_k"], out["mp_k_valid"] = mk, mkv
    builds = {
        "nulls": (np.arange(5, dtype=np.int64), np.zeros(5, dtype=bool)),
        "empty": (np.zeros(0, dtype=np.int64), np.zeros(0, dtype=bool)),
        "mixed": (np.array([1, 3, 5, 0, 7], dtype=np.int64), np.array([True, True, True, False, True])),
    }
    for name, (k, kv) in builds.items():
        con.load_table(f"mb_{name}", {"k": (k, kv)})
        r = con.execute(f"SELECT id, k IN (SELECT k FROM mb_{name}) FROM mp ORDER BY id")
        out[f"mb_{name}_k"], out[f"mb_{name}_k_valid"] = k, kv
        m, mv = col_arrays(r[1])
        out[f"mark_{name}"], out[f"mark_{name}_valid"] = np.where(mv, m, False).astype(bool), mv   # NULL rows: False
    con.execute("RESET disabled_optimizers")
    np.savez_compressed(os.path.join(OUT, "join_edge_cases.npz"), **out)


def _enum_values(path, enum_name):
    """{NAME: value} of `enum class <enum_name>` in a reference header (C rules: previous + 1 when not explicit)."""
    text = open(os.path.join(REF, path)).read()
    m = re.search(r"enum class " + enum_name + r"\b[^{]*\{(.*?)\};", text, re.S)
    assert m, f"{enum_name} not found in {path}"
    body = re.sub(r"//[^\n]*", "", m.group(1))
    values, nxt = {}, 0
    for item in body.split(","):
        m = re.match(r"\s*([A-Z_0-9]+)\s*(?:=\s*(\d+))?\s*$", item)
        if not m:
            continue
        nxt = int(m.group(2)) if m.group(2) is not None else nxt
        values[m.group(1)] = nxt
        nxt += 1
    return values


def _rows(rows):
    return [[py_scalar(x) for x in r] for r in rows]


def _summary(rows):
    """digest of a sorted row list + its length and first / last rows (they say where a mismatch is)"""
    rows = list(rows)
    return {"n": len(rows), "head": _rows(r if isinstance(r, (tuple, list)) else (r,) for r in rows[:3]),
            "tail": _rows(r if isinstance(r, (tuple, list)) else (r,) for r in rows[-3:]), "sha": digest(rows)}


def _column(values):
    v = np.asarray(values).astype(np.int64)
    return {"n": len(v), "head": v[:4].tolist(), "sha": digest_array(v)}


def reference_results(con):
    """The reference's answers for the tests that compare with it (tests/test_oracle.py, test_gpu_parity.py,
    test_gpu_reference_parity.py, test_bench_data.py, test_abi_layout.py).  Each input below is the one the test
    builds from the same seed or formula; large results are stored as a SHA-256 of their canonical row list
    (conftest.digest), small ones as rows."""
    import bench_data as BD

    out = {}
    # test_oracle.py: hash + group-by
    rng = np.random.default_rng(7)
    n = 4000
    k1 = rng.integers(-3, 3, size=n).astype(np.int32)
    k1v = rng.random(n) > 0.1
    k2 = rng.integers(0, 4, size=n).astype(np.uint8)
    x = rng.integers(-10 ** 12, 10 ** 12, size=n).astype(np.int64)
    xv = rng.random(n) > 0.2
    d = rng.standard_normal(n)
    con.load_table("pg", {"k1": (k1, k1v), "k2": k2, "x": (x, xv), "d": d})
    h = con.execute("SELECT hash(k1, k2) FROM pg")[0].values
    con.execute("SET perfect_ht_threshold=0")
    rows = con.fetchall("SELECT k1, k2, sum(x), count(x), count(*), min(x), max(x), avg(x), sum(d), min(d) "
                        "FROM pg GROUP BY k1, k2")
    con.execute("RESET perfect_ht_threshold")
    out["oracle_groupby"] = {"hash": digest_array(h), "rows": _rows(rows)}
    # test_oracle.py: joins
    rng = np.random.default_rng(11)
    nb, npr = 700, 1500
    bk = rng.integers(0, 200, size=nb).astype(np.int64)
    bkv = rng.random(nb) > 0.05
    bk2 = rng.integers(0, 3, size=nb).astype(np.int16)
    pk = rng.integers(0, 260, size=npr).astype(np.int64)
    pkv = rng.random(npr) > 0.05
    pk2 = rng.integers(0, 3, size=npr).astype(np.int16)
    con.load_table("jb", {"k": (bk, bkv), "k2": bk2, "id": np.arange(nb, dtype=np.int32)})
    con.load_table("jp", {"k": (pk, pkv), "k2": pk2, "id": np.arange(npr, dtype=np.int32)})
    joins = {}
    for name, keys_sql in (("k", "jp.k = jb.k"), ("k_k2", "jp.k = jb.k AND jp.k2 = jb.k2")):
        left = con.fetchall(f"SELECT jp.id, jb.id FROM jp LEFT JOIN jb ON {keys_sql}")
        joins[name] = {
            "inner": _summary(sorted(con.fetchall(f"SELECT jp.id, jb.id FROM jp JOIN jb ON {keys_sql}"))),
            "left": _summary(sorted((a, -1 if b is None else b) for a, b in left)),
            "semi": _summary(sorted(r[0] for r in con.fetchall(f"SELECT jp.id FROM jp SEMI JOIN jb ON {keys_sql}"))),
            "anti": _summary(sorted(r[0] for r in con.fetchall(f"SELECT jp.id FROM jp ANTI JOIN jb ON {keys_sql}"))),
        }
    mark = con.fetchall("SELECT id, k IN (SELECT k FROM jb) FROM jp ORDER BY id")
    joins["mark"] = _summary([(i, None if m is None else bool(m)) for i, m in mark])
    fb = np.array([0.0, np.nan, 1.5, -0.0, 2.5], dtype=np.float64)
    fp = np.array([-0.0, np.nan, 1.5, 7.0, np.nan], dtype=np.float64)
    con.load_table("fjb", {"k": fb, "id": np.arange(len(fb), dtype=np.int32)})
    con.load_table("fjp", {"k": fp, "id": np.arange(len(fp), dtype=np.int32)})
    joins["float_inner"] = _rows(sorted(con.fetchall("SELECT fjp.id, fjb.id FROM fjp JOIN fjb ON fjp.k = fjb.k")))
    out["oracle_joins"] = joins
    # test_oracle.py: filters
    rng = np.random.default_rng(13)
    n = 3000
    a = rng.integers(-5, 6, size=n).astype(np.int32)
    av = rng.random(n) > 0.15
    b = rng.integers(-5, 6, size=n).astype(np.int32)
    bv = rng.random(n) > 0.15
    f = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.5, -2.25]), size=n)
    fv = rng.random(n) > 0.1
    g = rng.choice(np.array([np.nan, np.inf, -0.0, 0.0, 1.5, 3.0]), size=n)
    con.load_table("fl", {"id": np.arange(n, dtype=np.int32), "a": (a, av), "b": (b, bv), "f": (f, fv), "g": g})
    sqls = ["a < b", "a = b OR a > 3", "a <> b AND b <= 3", "NOT (a >= b)", "a IS NULL OR b IS NOT NULL",
            "a IS DISTINCT FROM b", "a IS NOT DISTINCT FROM b", "(a < b) IS NULL", "NOT (a < b AND b < 3) OR a = 3",
            "f < g", "f >= g", "f = g", "f <> g", "f IS NOT DISTINCT FROM g", "f > 1.5::DOUBLE"]
    out["oracle_filters"] = {s: _summary(sorted(r[0] for r in con.fetchall(f"SELECT id FROM fl WHERE {s}")))
                             for s in sqls}
    # test_gpu_parity.py: group-by + join
    rng = np.random.default_rng(23)
    n = 200000
    k = rng.integers(0, 20000, size=n).astype(np.int64)
    x = rng.integers(-10 ** 9, 10 ** 9, size=n).astype(np.int64)
    d = rng.standard_normal(n)
    con.load_table("lr", {"k": k, "x": x, "d": d})
    con.execute("SET perfect_ht_threshold=0")
    rows = sorted(con.fetchall("SELECT k, sum(x), min(x), avg(d), count(*) FROM lr GROUP BY k"))
    con.execute("RESET perfect_ht_threshold")
    keys = np.array([r[0] for r in rows], dtype=np.int64)
    assert np.array_equal(keys, np.unique(k))
    ref_avg = np.array([r[3] for r in rows], dtype=np.float64)
    delta = ref_avg.view(np.uint64) - bincount_mean(k, d).view(np.uint64)   # mod 2^64: exact to undo
    small = delta.view(np.int64)
    assert np.abs(small).max() < 2 ** 31, "the bincount mean is too far from the reference to store compactly"
    np.savez_compressed(os.path.join(OUT, "reference_avg.npz"), ulp_delta=small.astype(np.int32))
    dim = np.unique(k)[::2].astype(np.int64)
    con.load_table("ld", {"k": dim, "p": (dim * 3).astype(np.int64)})
    out["gpu_live"] = {
        "groups": _summary([(r[0], r[1], r[2], r[4]) for r in rows]),
        "join": _rows([con.fetchall("SELECT count(*), sum(lr.x), sum(ld.p) FROM lr JOIN ld ON lr.k = ld.k")[0]])[0],
    }
    # test_gpu_reference_parity.py
    sf1 = 6_001_215
    con.execute(BD.q1_table_sql("q1in", sf1))
    out["sf1_q1"] = _rows(con.fetchall("SELECT rf, ls, sum(qty), sum(price), sum(disc_price), sum(charge), avg(qty), "
                                       "avg(price), avg(disc), count(*) FROM q1in GROUP BY rf, ls ORDER BY rf, ls"))
    con.execute("DROP TABLE q1in")
    con.execute(BD.probe_table_sql("li", sf1, 200_000))
    con.execute(BD.part_table_sql("part", 200_000))
    out["sf1_q14"] = _rows([con.fetchall("SELECT count(*), sum(price), sum(disc), sum(promo), sum(li.partkey * promo) "
                                         "FROM li JOIN part ON li.partkey = part.partkey")[0]])[0]
    con.execute("DROP TABLE li")
    con.execute("DROP TABLE part")
    card = {}
    for groups, n, keytypes in ((35, 3_000_000, "ssb"), (11_620, 3_000_000, "q3"), (3_500_000, 9_000_000, "q3")):
        if keytypes == "ssb":
            con.execute(BD.ssb_table_sql("t", n))
            sql = "SELECT year, nation, sum(profit), count(*) FROM t GROUP BY year, nation"
        else:
            con.execute(BD.q3_table_sql("t", n, groups))
            sql = "SELECT okey, odate, prio, sum(revenue), count(*) FROM t GROUP BY okey, odate, prio"
        rows = con.fetchall(sql)
        card[f"{keytypes}_{groups}_{n}"] = _summary(sorted(rows))
        con.execute("DROP TABLE t")
    out["sf1_groupby"] = card
    # test_bench_data.py: the synthetic columns as the reference's SQL defines them
    bench = {}

    def columns(sql):
        con.execute("DROP TABLE IF EXISTS t")
        con.execute(sql)
        return {c.name: _column(c.values) for c in con.execute("SELECT * FROM t")}

    for offset in (0, 591_855_000 * 3 + 12345):
        bench[f"q1_{offset}"] = columns(BD.q1_table_sql("t", 50_000, offset))
    n, nb, groups = 40_000, 1000, 5000
    bench["ssb"] = columns(BD.ssb_table_sql("t", n, 77))
    bench["q3"] = columns(BD.q3_table_sql("t", n, groups, 5))
    bench["probe"] = columns(BD.probe_table_sql("t", n, nb, 3))
    bench["part"] = columns(BD.part_table_sql("t", nb, 1001))
    bench["scan"] = columns(BD.scan_table_sql("t", n, 9))
    con.execute("DROP TABLE t")
    out["bench_data"] = bench
    # test_abi_layout.py: DuckDB's enum values the C ABI reuses
    out["enums"] = {
        "PhysicalType": _enum_values("src/include/duckdb/common/types.hpp", "PhysicalType"),
        "ExpressionType": _enum_values("src/include/duckdb/common/enums/expression_type.hpp", "ExpressionType"),
        "JoinType": _enum_values("src/include/duckdb/common/enums/join_type.hpp", "JoinType"),
        "VectorType": _enum_values("src/include/duckdb/common/enums/vector_type.hpp", "VectorType"),
    }
    with open(os.path.join(OUT, "reference_results.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True, separators=(",", ":"))
        fh.write("\n")


INT_NAMES = ["int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64"]


def _int_edges(name):
    """the limits of an integer type, +-1 around them and around 0, and the square-root and halving edges of MUL/ADD"""
    info = np.iinfo(name)
    lo, hi = int(info.min), int(info.max)
    r = int(np.sqrt(float(hi)))
    while (r + 1) * (r + 1) <= hi:
        r += 1
    while r * r > hi:
        r -= 1
    vals = {lo, lo + 1, -1, 0, 1, 2, hi // 2, hi // 2 + 1, r, r + 1, -r - 1, hi - 1, hi}
    return sorted(v for v in vals if lo <= v <= hi)


# integers whose conversion to FLOAT rounds differently when it goes through DOUBLE first, and integers near 2^53,
# 2^63 and 2^64 (UBIGINT values just below 2^64 round up to 2^64 as FLOAT)
ROUNDING_INTS = [2 ** 60 + 2 ** 36 + 1, 2 ** 60 + 2 ** 36, 2 ** 60 + 2 ** 36 - 1, 2 ** 53 + 1, 2 ** 53 - 1, 2 ** 24 + 1,
                 2 ** 62 + 2 ** 38 + 1, 2 ** 63 - 2 ** 39, 2 ** 63 - 2 ** 39 + 1, 2 ** 63, 2 ** 63 + 2 ** 39 + 1,
                 2 ** 64 - 2 ** 40 + 1, 2 ** 64 - 2 ** 39 - 1, 2 ** 64 - 2 ** 39, 2 ** 64 - 2 ** 39 + 1, 2 ** 64 - 2,
                 -(2 ** 60 + 2 ** 36 + 1), -(2 ** 53 + 1), -(2 ** 63 - 2 ** 39 + 1)]
FLT_MAX = float(np.finfo(np.float32).max)
# doubles at the FLOAT limits: FLT_MAX and the half-way point above it (which rounds to infinity), the smallest
# subnormals, a value that underflows to zero, and the non-finite values that pass through
DOUBLE_EDGES = [0.0, -0.0, 0.1, 1.5, -2.75, FLT_MAX, -FLT_MAX, 2.0 ** 128 - 2.0 ** 103, np.nextafter(2.0 ** 128 - 2.0 ** 103, 0),
                -(2.0 ** 128 - 2.0 ** 103), 2.0 ** 128, 1e300, -1e300, 2.0 ** -149, 2.0 ** -150, 3 * 2.0 ** -151, 1e-50,
                float("inf"), float("-inf"), float("nan"), 16777217.0, 1.0 + 2.0 ** -24 + 2.0 ** -52]
FLOAT_EDGES = [0.0, -0.0, 1.5, FLT_MAX, -FLT_MAX, 2.0 ** -149, float(np.float32(0.1)), float("inf"), float("-inf"),
               float("nan")]


def _enc(x, name):
    """a value of type `name` as JSON: integers exact, floats as float.hex (which keeps inf and nan)"""
    return float(x).hex() if name in ("float32", "float64") else (bool(x) if name == "bool" else int(x))


def _sql_lit(x, name):
    if name in ("float32", "float64"):
        return repr(float(x))
    return str(int(x))


def expr_edge_cases():
    """-> [{op, type, src?, args}]: every CAST pair among the integer types, integer -> FLOAT / DOUBLE / BOOLEAN,
    FLOAT -> DOUBLE and DOUBLE -> FLOAT, and ADD / SUB / MUL in every integer type, with operands at the edges"""
    cases = []
    for src in INT_NAMES:
        info = np.iinfo(src)
        for dst in INT_NAMES + ["bool", "float32", "float64"]:
            vals = set(_int_edges(src))
            if dst in INT_NAMES:
                d = np.iinfo(dst)
                vals |= {int(d.min) - 1, int(d.min), int(d.max), int(d.max) + 1}
            elif dst != "bool" and src in ("int64", "uint64"):
                vals |= set(ROUNDING_INTS)
            for x in sorted(v for v in vals if info.min <= v <= info.max):
                cases.append({"op": "cast", "src": src, "type": dst, "args": [x]})
    for x in FLOAT_EDGES:
        cases.append({"op": "cast", "src": "float32", "type": "float64", "args": [x]})
    for x in DOUBLE_EDGES:
        cases.append({"op": "cast", "src": "float64", "type": "float32", "args": [float(x)]})
    for t in INT_NAMES:
        edges = _int_edges(t)
        for op in ("add", "sub", "mul"):
            for a in edges:
                for b in edges:
                    cases.append({"op": op, "type": t, "args": [a, b]})
    return cases


def expr_cases(con):
    """expr_cases.json: DuckDB's result of every case of expr_edge_cases(), each in its own query, or "error" when the
    query fails with a conversion or overflow error"""
    sql_type = {np.dtype(k).name: v for k, v in R._SQL_OF_NP.items()}
    sym = {"add": "+", "sub": "-", "mul": "*"}
    out = []
    for case in expr_edge_cases():
        t = case["type"]
        if case["op"] == "cast":
            sql = f"SELECT CAST(CAST('{_sql_lit(case['args'][0], case['src'])}' AS {sql_type[case['src']]}) AS {sql_type[t]})"
        else:
            a, b = (f"CAST('{_sql_lit(x, t)}' AS {sql_type[t]})" for x in case["args"])
            sql = f"SELECT {a} {sym[case['op']]} {b}"
        try:
            col = con.execute(sql)[0]
            assert col.values.dtype == np.dtype(t), (sql, col.values.dtype)
            result = _enc(col.values[0], t)
        except RuntimeError as e:
            assert any(k in str(e) for k in ("Conversion Error", "Out of Range", "Overflow")), (sql, str(e))
            result = "error"
        out.append(dict(case, args=[_enc(x, case.get("src", t)) for x in case["args"]], result=result))
    with open(os.path.join(OUT, "expr_cases.json"), "w") as fh:
        json.dump(out, fh, separators=(",", ":"))
        fh.write("\n")


def main():
    """With arguments: only the named fixtures (e.g. `reference_results`), so that the others are not rewritten."""
    con = R.Connection(threads=4)
    for fn in sys.argv[1:] or ["hash_kat", "filter_cases", "join_cases", "tpch", "reference_results", "expr_cases",
                                     "join_edge_cases"]:
        globals()[fn](con)
    con.close()
    for f in sorted(os.listdir(OUT)):
        if f.endswith((".npz", ".json")):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
