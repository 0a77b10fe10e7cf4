"""The generic filter / projection path of filter.cu against exact references: the expression interpreter (eval_row in
filter_mask_kernel and compact_kernel), the three-launch tile-offset scan and the validity fill.

The interpreter runs every program the TMA tile path does not take: nullable columns, OR / NOT / IS [NOT] NULL /
[NOT] DISTINCT, FLOAT and DOUBLE, column-to-column comparisons, dictionary and constant vectors, arithmetic and CAST.
Each case compares the surviving count, out_sel, the mask bits (and the zero tail past n), and every projected value
and validity bit.  Integer references are exact (Python ints through oracle/port.py, whose CAST and checked arithmetic
are pinned to the reference's answers in tests/golden/expr_cases.json); FLOAT and DOUBLE results are compared bit for
bit (any NaN matches any NaN).  The kernel trace checks that the interpreter ran and the tile kernels did not."""
import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran, traced
from oracle import port as P
from test_gpu_parity import run_filter
from test_oracle import INT_NAMES, decode, expr_cases

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of filter.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "filter_mask_kernel": ["test_compare_all_types", "test_kleene_logic", "test_chains_at_the_limits",
                           "test_scan_three_chunks"],
    "compact_kernel": ["test_compare_all_types", "test_kleene_logic", "test_casts", "test_integer_arithmetic",
                       "test_scan_three_chunks"],
    "tile_scan_local_kernel": ["test_scan_three_chunks"],
    "tile_scan_chunks_kernel": ["test_scan_three_chunks"],
    "tile_scan_add_kernel": ["test_scan_three_chunks"],
    "fill_u64_kernel2": ["test_kleene_logic", "test_scan_three_chunks"],
}
# kernels of filter.cu that no test here has to reach, with the reason
KERNEL_EXCLUDED = {}

TILE_KERNELS = ("filter_mask_tile_kernel", "compact_tile_kernel", "filter_fused_tile_kernel")
CMP_OPS = ["eq", "ne", "lt", "gt", "le", "ge", "distinct", "notdistinct"]
ALL_DTYPES = [np.bool_, np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64, np.float32,
              np.float64]


def edges(dtype):
    """values at the limits of a type: MIN, MIN+1, -1, 0, 1, MAX-1, MAX (UBIGINT also both sides of 2^63); for
    FLOAT / DOUBLE +-0, +-inf, NaN, the largest and the smallest subnormal values"""
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return np.array([False, True])
    if dt.kind == "f":
        fi = np.finfo(dt)
        return np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.5, -1.5, fi.max, -fi.max, fi.smallest_subnormal,
                         -fi.smallest_subnormal], dtype=dt)
    info = np.iinfo(dt)
    vals = {int(info.min), int(info.min) + 1, 0, 1, int(info.max) - 1, int(info.max)}
    if dt.kind == "i":
        vals.add(-1)
    if dt == np.uint64:
        vals |= {2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1}
    return np.array(sorted(vals), dtype=dt)


def assert_same(got, exp, what=""):
    """bit-exact equality; any NaN matches any NaN"""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (what, got.dtype, exp.dtype, got.shape, exp.shape)
    if exp.dtype.kind == "f":
        gn, en = np.isnan(got), np.isnan(exp)
        np.testing.assert_array_equal(gn, en, err_msg=str(what))
        got, exp = got[~gn], exp[~en]
        got, exp = got.view(f"u{exp.itemsize}"), exp.view(f"u{exp.itemsize}")
    np.testing.assert_array_equal(got, exp, err_msg=str(what))


def check(ctx, vectors, cols, n, pred, projs=()):
    """run the program; compare count, out_sel, mask (with its zero tail) and the projected values and validity with
    the oracle.  Projections are evaluated on the surviving rows only, as DuckDB's projection above the filter does."""
    if pred is None:
        exp_sel, keep = np.arange(n, dtype=np.uint32), np.ones(n, dtype=bool)
    else:
        exp_sel, keep = P.filter_select(pred, cols, n)
    count, sel, mask, outs = run_filter(ctx, None, n, pred, projs, vectors=vectors)
    assert count == len(exp_sel), (pred, count, len(exp_sel))
    np.testing.assert_array_equal(sel, exp_sel, err_msg=str(pred))
    if pred is not None and n:
        np.testing.assert_array_equal(capi.valid_from_words(mask, n), keep, err_msg=str(pred))
        if n % 64:
            assert int(mask[-1]) >> (n % 64) == 0, pred
    kept = [(v[exp_sel], valid[exp_sel] if valid is not None else None) for v, valid in cols]
    for (v, valid), p in zip(outs, projs):
        ev, evalid = P.eval_expr(p, kept, len(exp_sel))
        np.testing.assert_array_equal(valid, evalid, err_msg=str(p))
        assert_same(v[valid], ev.astype(v.dtype)[evalid], p)
    return count


# ------------------------------------------------------------------ comparisons
@pytest.mark.parametrize("dtype", ALL_DTYPES, ids=lambda d: np.dtype(d).name)
def test_compare_all_types(ctx, dtype):
    """The six comparisons and [NOT] DISTINCT FROM, column-column and column-constant in both orders, over every type:
    every pair of edge values, NULLs on either side, a dictionary column with dictionary-indexed validity, a constant
    vector, a NULL constant vector and a NULL constant node.  The comparison is also projected as a BOOL column."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(dt.num)
    e = edges(dt)
    k = len(e)
    a = np.concatenate([np.repeat(e, k), rng.choice(e, 300)]).astype(dt)
    b = np.concatenate([np.tile(e, k), rng.choice(e, 300)]).astype(dt)
    n = len(a)
    av, bv = rng.random(n) > 0.15, rng.random(n) > 0.15
    dv = np.arange(k) % 4 != 3  # dictionary validity, by dictionary position
    dsel = rng.integers(0, k, size=n).astype(np.uint32)
    const = e[k // 2]
    vectors = [ops.Vector.flat(a, av), ops.Vector.flat(b, bv), ops.Vector.dictionary(e, dsel, dv),
               ops.Vector.constant(const, dt), ops.Vector.constant(const, dt, is_null=True), ops.Vector.flat(a)]
    cols = [(a, av), (b, bv), (e[dsel], dv[dsel]), (np.full(n, const, dtype=dt), None),
            (np.zeros(n, dtype=dt), np.zeros(n, dtype=bool)), (a, None)]
    c = lambda i: ("col", i)  # noqa: E731
    # (column 5, the flat column without validity, only meets other columns: against a constant the tile path takes it)
    shapes = [(c(0), c(1)), (c(1), c(0)), (c(5), c(2)), (c(2), c(0)), (c(0), c(3)), (c(3), c(1)), (c(4), c(0)),
              (c(5), c(4))]
    for x in e:
        shapes += [(c(0), ("const", x, dt)), (("const", x, dt), c(0)), (c(2), ("const", x, dt))]
    shapes += [(c(0), ("const", 0, dt, True)), (("const", 0, dt, True), c(1))]

    def run():
        for op in CMP_OPS:
            for lhs, rhs in shapes:
                pred = (op, lhs, rhs)
                check(ctx, vectors, cols, n, pred, [pred, c(0)])

    _, names = traced(run)
    assert_ran(names, "filter_mask_kernel", "compact_kernel<false>")
    assert_not_ran(names, *TILE_KERNELS)


# ------------------------------------------------------------------ three-valued logic
def test_kleene_logic(ctx):
    """AND, OR, NOT, IS NULL and IS NOT NULL over every pair from {TRUE, FALSE, NULL}, as the filter and as projected
    BOOL columns (a projection-only program runs compact_kernel<true>)."""
    tv = np.array([1, 0, 0], dtype=bool)          # TRUE, FALSE, NULL (its stored value is arbitrary: 0 and 1 below)
    vv = np.array([True, True, False])
    reps = 700
    p = np.tile(np.repeat(tv, 3), reps)
    q = np.tile(np.tile(tv, 3), reps)
    pv = np.tile(np.repeat(vv, 3), reps)
    qv = np.tile(np.tile(vv, 3), reps)
    n = len(p)
    p[::2] |= ~pv[::2]                                # NULLs that store 1 as well as 0
    cols = [(p, pv), (q, qv)]
    vectors = [ops.Vector.flat(p, pv), ops.Vector.flat(q, qv)]
    c = lambda i: ("col", i)  # noqa: E731
    exprs = [("and", c(0), c(1)), ("or", c(0), c(1)), ("not", c(0)), ("isnull", c(0)), ("isnotnull", c(1)),
             ("not", ("and", c(0), c(1))), ("or", ("not", c(0)), ("isnull", c(1))),
             ("and", ("or", c(0), c(1)), ("not", c(1))), ("isnull", ("and", c(0), c(1))),
             ("isnotnull", ("or", c(0), c(1)))]

    def run():
        for x in exprs:
            check(ctx, vectors, cols, n, x, [x, c(0)])
            check(ctx, vectors, cols, n, None, exprs[:6] + [x])

    _, names = traced(run)
    assert_ran(names, "filter_mask_kernel", "compact_kernel<false>", "compact_kernel<true>", "fill_u64_kernel2")
    assert_not_ran(names, *TILE_KERNELS)


def left_deep(op, terms):
    t = terms[0]
    for x in terms[1:]:
        t = (op, t, x)
    return t


def node_count(t):
    return 1 + sum(node_count(x) for x in t[1:] if isinstance(x, tuple))


# twelve columns in pairs of one type, and a thirteenth
CHAIN_DTYPES = [np.int8, np.int8, np.uint16, np.uint16, np.int32, np.int32, np.uint64, np.uint64, np.float32,
                np.float32, np.float64, np.float64, np.bool_]


def test_chains_at_the_limits(ctx):
    """Left-deep AND / OR chains as the DuckDB binding builds them, up to 24 nodes and 12 distinct columns, with 12
    projections.  One more node, projection or distinct column returns B200_ERR_INVALID."""
    rng = np.random.default_rng(5)
    n = 5003
    cols, vectors = [], []
    for dt in CHAIN_DTYPES:
        e = edges(dt)
        v = rng.choice(e, n).astype(dt)
        valid = rng.random(n) > 0.1
        cols.append((v, valid))
        vectors.append(ops.Vector.flat(v, valid))
    c = lambda i: ("col", i)  # noqa: E731
    ops_ = ["lt", "ge", "ne", "distinct", "le", "gt"]
    # six column-column terms over twelve distinct columns (pairs of equal type), one negated: 24 nodes
    col_terms = [(o, c(2 * j), c(2 * j + 1)) for j, o in enumerate(ops_)]
    col_terms[3] = ("not", col_terms[3])
    # six column-constant terms: 23 nodes, and the NOT makes 24
    const_terms = [(o, c(2 * j), ("const", edges(CHAIN_DTYPES[2 * j])[1], np.dtype(CHAIN_DTYPES[2 * j])))
                   for j, o in enumerate(ops_)]
    const_terms[2] = ("not", const_terms[2])

    def run():
        counts = []
        for terms in (col_terms, const_terms):
            for op in ("and", "or"):
                for k in range(1, 7):
                    pred = left_deep(op, terms[:k])
                    counts.append(check(ctx, vectors, cols, n, pred))
                assert node_count(pred) == 24
        # 12 projections of 12 distinct columns next to a 3-node filter
        pred = ("lt", c(0), ("const", 0, np.int8))
        check(ctx, vectors, cols, n, pred, [c(i) for i in range(12)])
        return counts

    counts, names = traced(run)
    assert_ran(names, "filter_mask_kernel")
    assert_not_ran(names, *TILE_KERNELS)
    assert min(counts) < n // 2 < max(counts)

    def invalid(pred, projs):
        with pytest.raises(capi.B200Error) as err:
            run_filter(ctx, None, n, pred, projs, vectors=vectors)
        assert err.value.code == capi.ERR_INVALID, (pred, projs)

    invalid(("not", left_deep("and", col_terms)), [])                                   # 25 nodes
    invalid(("lt", c(0), ("const", 0, np.int8)), [c(i % 12) for i in range(13)])        # 13 projections
    invalid(("lt", c(0), ("const", 0, np.int8)), [c(i) for i in range(1, 13)])         # 13 distinct columns
    invalid(left_deep("or", col_terms), [c(12)])                                         # 13 distinct columns


# ------------------------------------------------------------------ CAST
def cast_groups():
    groups = {}
    for case in expr_cases():
        if case["op"] == "cast":
            groups.setdefault((case["src"], case["type"]), []).append(case)
    return groups


@pytest.mark.parametrize("source", INT_NAMES + ["float32", "float64"])
def test_casts(ctx, source):
    """Every CAST of the reference's edge cases from one source type: the values that convert are projected in one
    column and must equal the reference's results bit for bit; each value the reference refuses must make the call fail
    with B200_ERR_OVERFLOW, and must not when it is NULL or when the filter drops its row."""
    groups = {k: v for k, v in cast_groups().items() if k[0] == source}
    assert len(groups) == (11 if source in INT_NAMES else 1)

    def run():
        nerr = 0
        for (src, dst), cases in sorted(groups.items()):
            sdt, ddt = np.dtype(src), np.dtype(dst)
            good = [c for c in cases if c["result"] != "error"]
            bad = [c for c in cases if c["result"] == "error"]
            x = np.array([decode(c["args"][0], src) for c in good], dtype=sdt)
            exp = np.array([decode(c["result"], dst) for c in good], dtype=ddt)
            count, _, _, outs = run_filter(ctx, None, len(x), None, [("cast", ddt, ("col", 0))],
                                           vectors=[ops.Vector.flat(x)])
            assert count == len(x)
            assert_same(outs[0][0], exp, (src, dst))
            for c in bad:
                v = np.array([decode(c["args"][0], src)] * 3, dtype=sdt)
                with pytest.raises(capi.B200Error) as err:
                    run_filter(ctx, None, 3, None, [("cast", ddt, ("col", 0))], vectors=[ops.Vector.flat(v)])
                assert err.value.code == capi.ERR_OVERFLOW, c
                # the same node in a comparison fails too
                with pytest.raises(capi.B200Error) as err:
                    run_filter(ctx, None, 3, ("eq", ("cast", ddt, ("col", 0)), ("cast", ddt, ("col", 0))), [],
                               vectors=[ops.Vector.flat(v, np.array([False, True, False]))])
                assert err.value.code == capi.ERR_OVERFLOW, c
                nerr += 1
            if bad:
                # refused values in NULL rows and in rows the filter drops do not raise
                v = np.array([decode(c["args"][0], src) for c in bad] + [0], dtype=sdt)
                m = len(v)
                valid = np.zeros(m, dtype=bool)
                valid[-1] = True
                count, _, _, outs = run_filter(ctx, None, m, None, [("cast", ddt, ("col", 0))],
                                               vectors=[ops.Vector.flat(v, valid)])
                np.testing.assert_array_equal(outs[0][1], valid)
                drop = np.arange(m) == m - 1
                count, sel, _, outs = run_filter(ctx, None, m, ("col", 1), [("cast", ddt, ("col", 0))],
                                                 vectors=[ops.Vector.flat(v), ops.Vector.flat(drop)])
                assert count == 1 and sel.tolist() == [m - 1]
                assert_same(outs[0][0], np.zeros(1, dtype=ddt))
        return nerr

    nerr, names = traced(run)
    assert nerr > 0 or source == "float32"
    assert_ran(names, "compact_kernel<true>")
    if nerr:
        assert_ran(names, "compact_kernel<false>", "filter_mask_kernel")
    assert_not_ran(names, *TILE_KERNELS)


def test_float_to_integer_cast_rejected(ctx):
    """FLOAT / DOUBLE -> integer is not implemented (the bits used to be read as the integer): B200_ERR_INVALID"""
    for src in (np.float32, np.float64):
        for dst in (np.int8, np.uint64, np.int64, np.bool_):
            v = np.ones(4, dtype=src)
            with pytest.raises(capi.B200Error) as err:
                run_filter(ctx, None, 4, None, [("cast", np.dtype(dst), ("col", 0))], vectors=[ops.Vector.flat(v)])
            assert err.value.code == capi.ERR_INVALID


def test_cast_rounds_once_to_float(ctx):
    """BIGINT / UBIGINT -> FLOAT rounds once, like static_cast<float>: 2^60 + 2^36 + 1 becomes 2^60 + 2^37 (through
    DOUBLE it would be 2^60), and UBIGINT values in (2^64 - 2^39, 2^64) become 2^64."""
    rng = np.random.default_rng(9)
    m = 20000
    for dt in (np.int64, np.uint64):
        info = np.iinfo(dt)
        x = rng.integers(info.min, info.max, size=m, dtype=dt, endpoint=True)
        # a FLOAT (24-bit significand at 2^e) plus half its ulp plus or minus a little: exactly representable
        # only in 64 bits, a half-way case in DOUBLE, so rounding through DOUBLE goes the wrong way for half of them
        e = rng.integers(54, 63 if dt == np.int64 else 64, size=m)
        sig = rng.integers(2 ** 23, 2 ** 24, size=m)
        near = [(int(s) << (int(k) - 23)) + (1 << (int(k) - 24)) + int(d)
                for s, k, d in zip(sig, e, rng.choice([-2, -1, 1, 2], size=m))]
        near = np.array([v if v < 2 ** 64 else v - 4 for v in near], dtype=object)
        near = near.astype(np.uint64) if dt == np.uint64 else \
            np.array([v if v < 2 ** 63 else v - 2 ** 63 for v in near], dtype=object).astype(np.int64)
        if dt == np.int64:
            near[::2] = -near[::2]
        v = np.concatenate([x, near.astype(dt)])
        count, _, _, outs = run_filter(ctx, None, len(v), None, [("cast", np.dtype(np.float32), ("col", 0))],
                                       vectors=[ops.Vector.flat(v)])
        assert_same(outs[0][0], v.astype(np.float32), dt)
    assert int(np.float32(np.int64(2 ** 60 + 2 ** 36 + 1))) == 2 ** 60 + 2 ** 37


# ------------------------------------------------------------------ arithmetic
def arith_groups():
    groups = {}
    for case in expr_cases():
        if case["op"] != "cast":
            groups.setdefault((case["op"], case["type"]), []).append(case)
    return groups


OPS = {"add": capi.EXPR_ADD, "sub": capi.EXPR_SUB, "mul": capi.EXPR_MUL}


@pytest.mark.parametrize("tname", INT_NAMES)
def test_integer_arithmetic(ctx, tname):
    """ADD, SUB and MUL with every pair of edge operands of the reference's cases:
    - checked (mode 1): the results the reference computes, bit for bit, and B200_ERR_OVERFLOW for each pair it
      refuses, but not when an operand is NULL or when the filter drops the row;
    - unchecked (mode 0): the result wraps to the type, stored and compared (`(a op b) < 0` and `= const`);
    - DECIMAL (mode 2, INT16 / INT32 / INT64): the port's answer at the DECIMAL bounds."""
    dt = np.dtype(tname)
    groups = arith_groups()
    c = lambda i: ("col", i)  # noqa: E731

    def run():
        for op in OPS:
            cases = groups[(op, tname)]
            a = np.array([int(x["args"][0]) for x in cases], dtype=object).astype(dt)
            b = np.array([int(x["args"][1]) for x in cases], dtype=object).astype(dt)
            err = np.array([x["result"] == "error" for x in cases])
            n = len(cases)
            expr = (op, dt, c(0), c(1), 1)
            # rows the reference computes: one column
            ok = ~err
            count, _, _, outs = run_filter(ctx, None, int(ok.sum()), None, [expr],
                                           vectors=[ops.Vector.flat(a[ok]), ops.Vector.flat(b[ok])])
            exp = np.array([int(x["result"]) for x, e in zip(cases, err) if not e], dtype=object).astype(dt)
            assert_same(outs[0][0], exp, (op, tname))
            # each refused pair fails alone, as a projection and inside a filter
            for i in np.nonzero(err)[0]:
                for pred, projs in ((None, [expr]), (("lt", expr, ("const", 0, dt)), [])):
                    with pytest.raises(capi.B200Error) as e:
                        run_filter(ctx, None, 1, pred, projs, vectors=[ops.Vector.flat(a[i:i + 1]),
                                                                       ops.Vector.flat(b[i:i + 1])])
                    assert e.value.code == capi.ERR_OVERFLOW, cases[i]
            # ... but not with a NULL operand, nor in rows the filter drops
            rng = np.random.default_rng(len(cases))
            side = rng.random(n) < 0.5
            av, bv = ~(err & side), ~(err & ~side)
            check(ctx, [ops.Vector.flat(a, av), ops.Vector.flat(b, bv)], [(a, av), (b, bv)], n, None, [expr])
            check(ctx, [ops.Vector.flat(a), ops.Vector.flat(b), ops.Vector.flat(~err)],
                  [(a, None), (b, None), (~err, None)], n, c(2), [expr, c(0)])
            # unchecked: wraps, and the wrapped value is what a comparison sees
            wrap = (op, dt, c(0), c(1), 0)
            vec = [ops.Vector.flat(a, av), ops.Vector.flat(b)]
            cl = [(a, av), (b, None)]
            check(ctx, vec, cl, n, ("lt", wrap, ("const", 0, dt)), [wrap])
            check(ctx, vec, cl, n, ("ge", wrap, ("const", 1, dt)), [wrap, c(1)])
            check(ctx, vec, cl, n, ("eq", wrap, ("const", int(np.iinfo(dt).max), dt)), [])
            check(ctx, vec, cl, n, None, [wrap, (op, dt, wrap, c(1), 0)])
            if tname in ("int16", "int32", "int64"):
                bound = {"int16": 9999, "int32": 999999999, "int64": 10 ** 18 - 1}[tname]
                ops_ = [bound, bound - 1, 1, 0, -1, -bound, -bound + 1, 2, int(np.sqrt(bound)), int(np.sqrt(bound)) + 1]
                x = np.array([p for p in ops_ for _ in ops_], dtype=dt)
                y = np.array([q for _ in ops_ for q in ops_], dtype=dt)
                dec = (op, dt, c(0), c(1), 2)
                exact = [int(p) + int(q) if op == "add" else int(p) - int(q) if op == "sub" else int(p) * int(q)
                         for p, q in zip(x, y)]
                bad = np.array([abs(v) > bound for v in exact])
                assert bad.any() and not bad.all()
                check(ctx, [ops.Vector.flat(x[~bad]), ops.Vector.flat(y[~bad])], [(x[~bad], None), (y[~bad], None)],
                      int((~bad).sum()), None, [dec])
                for i in np.nonzero(bad)[0]:
                    with pytest.raises(capi.B200Error) as e:
                        run_filter(ctx, None, 1, None, [dec], vectors=[ops.Vector.flat(x[i:i + 1]),
                                                                       ops.Vector.flat(y[i:i + 1])])
                    assert e.value.code == capi.ERR_OVERFLOW, (op, x[i], y[i])

    _, names = traced(run)
    assert_ran(names, "compact_kernel<true>", "compact_kernel<false>", "filter_mask_kernel")
    assert_not_ran(names, *TILE_KERNELS)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["float32", "float64"])
def test_float_arithmetic(ctx, dtype):
    """FLOAT and DOUBLE + - * on every pair of edge values (+-0, +-inf, NaN, MAX, subnormals) and random values, bit
    for bit against numpy in the same width: the FLOAT results are rounded once."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(dt.itemsize)
    e = edges(dt)
    r = (rng.standard_normal(5000) * 10.0 ** rng.integers(-30, 30, size=5000)).astype(dt)
    a = np.concatenate([np.repeat(e, len(e)), r, r[::-1]]).astype(dt)
    b = np.concatenate([np.tile(e, len(e)), r[::-1] * dt.type(3.25), r]).astype(dt)
    n = len(a)
    valid = rng.random(n) > 0.05
    c = lambda i: ("col", i)  # noqa: E731
    for op in OPS:
        for m in (0, 1):
            check(ctx, [ops.Vector.flat(a, valid), ops.Vector.flat(b)], [(a, valid), (b, None)], n,
                  ("ne", (op, dt, c(0), c(1), m), ("const", 0.0, dt)), [(op, dt, c(0), c(1), m), c(0)])


def test_arithmetic_operand_types_rejected(ctx):
    """ADD / SUB / MUL whose operands do not both have the node's type, on BOOL, or with a check mode outside 0..2
    (2 outside INT16 / INT32 / INT64) return B200_ERR_INVALID: a FLOAT operand under a DOUBLE ADD used to be read as
    a double."""
    n = 100
    f, d = np.ones(n, dtype=np.float32), np.ones(n, dtype=np.float64)
    i8, i64, u32 = np.ones(n, dtype=np.int8), np.ones(n, dtype=np.int64), np.ones(n, dtype=np.uint32)
    bo = np.ones(n, dtype=bool)
    c = lambda i: ("col", i)  # noqa: E731
    for vec, expr in [([f, d], ("add", np.dtype(np.float64), c(0), c(1))),
                      ([d, f], ("mul", np.dtype(np.float32), c(0), c(1))),
                      ([i8, i64], ("sub", np.dtype(np.int64), c(1), c(0))),
                      ([i64, i64], ("add", np.dtype(np.int32), c(0), c(1))),
                      ([bo, bo], ("add", np.dtype(np.bool_), c(0), c(1), 0)),
                      ([u32, u32], ("mul", np.dtype(np.uint32), c(0), c(1), 2)),
                      ([i64, i64], ("mul", np.dtype(np.int64), c(0), c(1), 3))]:
        with pytest.raises(capi.B200Error) as err:
            run_filter(ctx, None, n, None, [expr], vectors=[ops.Vector.flat(v) for v in vec])
        assert err.value.code == capi.ERR_INVALID, expr
    # a matching program runs
    run_filter(ctx, None, n, None, [("add", np.dtype(np.float32), c(0), ("cast", np.dtype(np.float32), c(1)))],
               vectors=[ops.Vector.flat(f), ops.Vector.flat(i8)])


# ------------------------------------------------------------------ scan
SCAN_N = 2 * 8_388_608 + 5 * 2048 + 37  # three 4096-tile chunks, the last one partial, ending in a partial tile


def test_scan_three_chunks(ctx):
    """A 1-byte column long enough for three chunks of the tile-offset scan: the interpreter's mask and compaction
    (nullable column) and the tile mask kernel (flat column) both feed it, with and without a projection."""
    rng = np.random.default_rng(17)
    n = SCAN_N
    # survivor density varies across the chunks so that a wrong chunk base shifts the output
    x = rng.integers(0, 256, size=n, dtype=np.uint8)
    x[: n // 3] //= 2
    valid = rng.random(n) > 0.05
    c = lambda i: ("col", i)  # noqa: E731
    pred = ("lt", c(0), ("const", 100, np.uint8))
    for nullable in (True, False):
        vectors = [ops.Vector.flat(x, valid if nullable else None)]
        cols = [(x, valid if nullable else None)]
        for projs in ([c(0)], []):
            def run():
                return check(ctx, vectors, cols, n, pred, projs)

            count, names = traced(run)
            assert n // 4 < count < 3 * n // 4
            assert_ran(names, "tile_scan_local_kernel", "tile_scan_chunks_kernel", "tile_scan_add_kernel")
            if nullable:
                assert_ran(names, "filter_mask_kernel", "compact_kernel<false>")
                if projs:
                    assert_ran(names, "fill_u64_kernel2")
                assert_not_ran(names, *TILE_KERNELS)
            else:
                assert_ran(names, "filter_mask_tile_kernel")
                assert_ran(names, "compact_tile_kernel" if projs else "compact_kernel<false>")
                assert_not_ran(names, "filter_mask_kernel")
