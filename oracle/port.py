"""CPU restatement (numpy) of the reference's algorithms on the hot path.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg - never by the product package duckdb_b200.

Parity status: PINNED.  Every function below is checked in tests/test_oracle.py
against (a) the reference's own known-answer vectors
(test/sql/function/generic/hash_func.test:22,160-171), (b) golden fixtures in
tests/golden/ produced by running the unmodified reference
(oracle/_ref/libduckdb_ref.so, script tests/golden/make_golden.py), and (c) -
when oracle/_ref is present - live against the reference on random inputs.

Columns are (values ndarray, valid bool ndarray | None).
"""
import numpy as np

U64 = np.uint64
_M = U64(0xD6E8FEB86659FD93)
NULL_HASH = U64(0xBF58476D1CE4E5B9)  # vector_hash.cpp:23 HashOp::NULL_HASH


def murmur64(x):
    """duckdb::MurmurHash64 (src/include/duckdb/common/types/hash.hpp:38-45)."""
    x = np.asarray(x, dtype=U64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> U64(32)
        x *= _M
        x ^= x >> U64(32)
        x *= _M
        x ^= x >> U64(32)
    return x


_MASK64 = (1 << 64) - 1
_M_INV = pow(0xD6E8FEB86659FD93, -1, 1 << 64)


def murmur64_inverse(h):
    """the 64-bit word x with murmur64(x) == h (Python ints).  Each step of murmur64 is a bijection: the xor-shift by 32
    is its own inverse and the odd multiplier has an inverse modulo 2^64."""
    x = int(h) & _MASK64
    x ^= x >> 32
    x = (x * _M_INV) & _MASK64
    x ^= x >> 32
    x = (x * _M_INV) & _MASK64
    x ^= x >> 32
    return x


def combine_hash_preimage(prefix_hash, target):
    """the BIGINT / UBIGINT key bits b (Python int) that give combine_hash(prefix_hash, murmur64(b)) == target: lets a test
    give two different composite keys the same 64-bit hash, or a composite key any hash it wants"""
    a = int(prefix_hash) & _MASK64
    a ^= a >> 32
    a = (a * int(_M)) & _MASK64
    return murmur64_inverse((int(target) & _MASK64) ^ a)


def hash_values(values):
    """duckdb::Hash<T> (hash.hpp:47-54, hash.cpp:33-57): ints < 64 bit hash their uint32 cast;
    floats: -0.0 -> +0.0 and NaN -> canonical quiet NaN, then the raw bits."""
    v = np.asarray(values)
    if v.dtype == np.float64:
        w = v.copy()
        w[w == 0.0] = 0.0
        bits = w.view(U64).copy()
        bits[np.isnan(w)] = U64(0x7FF8000000000000)
        return murmur64(bits)
    if v.dtype == np.float32:
        w = v.copy()
        w[w == 0.0] = 0.0
        bits = w.view(np.uint32).copy()
        bits[np.isnan(w)] = np.uint32(0x7FC00000)
        return murmur64(bits.astype(U64))
    if v.dtype in (np.dtype(np.int64), np.dtype(np.uint64)):
        return murmur64(v.view(U64) if v.dtype == np.int64 else v)
    if v.dtype == np.bool_:
        return murmur64(v.astype(U64))
    # static_cast<uint32_t>(value): sign-extend to 32 bits, reinterpret
    return murmur64(v.astype(np.int64).astype(np.uint32).astype(U64) if v.dtype.kind == "i"
                    else v.astype(np.uint32).astype(U64))


def combine_hash(a, b):
    """CombineHashScalar (vector_hash.cpp:44-48)."""
    a = np.asarray(a, dtype=U64).copy()
    with np.errstate(over="ignore"):
        a ^= a >> U64(32)
        a *= _M
    return a ^ np.asarray(b, dtype=U64)


def hash_columns(cols):
    """VectorOperations::Hash then CombineHash per further column (vector_hash.cpp:504-552);
    NULL hashes to NULL_HASH."""
    h = None
    for values, valid in cols:
        hv = hash_values(values)
        if valid is not None:
            hv = np.where(valid, hv, NULL_HASH)
        h = hv if h is None else combine_hash(h, hv)
    return h


def radix_partition_ids(hashes, bits):
    """RadixPartitioning::ApplyMask (radix_partitioning.hpp:45-61): (hash >> (48-bits)) & (2^bits-1)."""
    if bits == 0:
        return np.zeros(len(hashes), dtype=np.uint32)
    return ((np.asarray(hashes, dtype=U64) >> U64(48 - bits)) & U64((1 << bits) - 1)).astype(np.uint32)


# ------------------------------------------------------------------ filter / projection
def _cmp3(a, b):
    """three-way compare with DuckDB's float total order (comparison_operators.cpp:24-90)."""
    if a.dtype.kind == "f":
        an, bn = np.isnan(a), np.isnan(b)
        with np.errstate(invalid="ignore"):
            c = np.where(a < b, -1, np.where(a > b, 1, 0))
        c = np.where(an & bn, 0, np.where(an, 1, np.where(bn, -1, c)))
        return c
    return np.where(a < b, -1, np.where(a > b, 1, 0))


_INT_RANGE = {
    np.dtype(np.int8): (-128, 127), np.dtype(np.int16): (-32768, 32767),
    np.dtype(np.int32): (-2 ** 31, 2 ** 31 - 1), np.dtype(np.int64): (-2 ** 63, 2 ** 63 - 1),
    np.dtype(np.uint8): (0, 255), np.dtype(np.uint16): (0, 65535), np.dtype(np.uint32): (0, 2 ** 32 - 1),
    np.dtype(np.uint64): (0, 2 ** 64 - 1),
}
_DEC_RANGE = {np.dtype(np.int16): 9999, np.dtype(np.int32): 999999999, np.dtype(np.int64): 999999999999999999}


class OverflowError_(Exception):
    pass


def eval_expr(node, cols, n):
    """Evaluate an expression tree -> (values, valid).  node is a tuple:
    ('col', i) | ('const', value, dtype, is_null) | (cmp, l, r) with cmp in eq ne lt gt le ge distinct notdistinct |
    ('and', l, r) | ('or', l, r) | ('not', c) | ('isnull', c) | ('isnotnull', c) |
    ('add'|'sub'|'mul', dtype, l, r, check_mode) | ('cast', dtype, c).
    Semantics: ExpressionExecutor (expression_executor.cpp:253-307), NULL handling
    comparison_operators.hpp:199-229, AND/OR three-valued logic (boolean_operators.cpp)."""
    op = node[0]
    if op == "col":
        v, valid = cols[node[1]]
        return v, (np.ones(n, dtype=bool) if valid is None else valid)
    if op == "const":
        dt = np.dtype(node[2])
        isnull = len(node) > 3 and node[3]
        return np.full(n, 0 if isnull else node[1], dtype=dt), np.full(n, not isnull, dtype=bool)
    if op in ("eq", "ne", "lt", "gt", "le", "ge"):
        a, av = eval_expr(node[1], cols, n)
        b, bv = eval_expr(node[2], cols, n)
        c = _cmp3(a, b)
        r = {"eq": c == 0, "ne": c != 0, "lt": c < 0, "gt": c > 0, "le": c <= 0, "ge": c >= 0}[op]
        return r, av & bv
    if op in ("distinct", "notdistinct"):
        a, av = eval_expr(node[1], cols, n)
        b, bv = eval_expr(node[2], cols, n)
        d = np.where(av & bv, _cmp3(a, b) != 0, av != bv)
        return (d if op == "distinct" else ~d), np.ones(n, dtype=bool)
    if op in ("and", "or"):
        a, av = eval_expr(node[1], cols, n)
        b, bv = eval_expr(node[2], cols, n)
        a, b = a.astype(bool), b.astype(bool)
        if op == "and":
            is_false = (av & ~a) | (bv & ~b)
            valid = is_false | (av & bv)
            return np.where(is_false, False, True) & valid, valid
        is_true = (av & a) | (bv & b)
        valid = is_true | (av & bv)
        return is_true, valid
    if op == "not":
        a, av = eval_expr(node[1], cols, n)
        return ~a.astype(bool), av
    if op == "isnull":
        _, av = eval_expr(node[1], cols, n)
        return ~av, np.ones(n, dtype=bool)
    if op == "isnotnull":
        _, av = eval_expr(node[1], cols, n)
        return av.copy(), np.ones(n, dtype=bool)
    if op in ("add", "sub", "mul"):
        dt = np.dtype(node[1])
        a, av = eval_expr(node[2], cols, n)
        b, bv = eval_expr(node[3], cols, n)
        mode = node[4] if len(node) > 4 else 1
        valid = av & bv
        if dt.kind == "f":
            with np.errstate(all="ignore"):
                r = {"add": a + b, "sub": a - b, "mul": a * b}[op].astype(dt)
            return r, valid
        # exact python-int arithmetic, then the overflow rule of the result type
        # (TryAddOperator / TryDecimalAdd, add.cpp:260; TryDecimalMultiply multiply.cpp:299)
        ea = a.astype(object)
        eb = b.astype(object)
        r = {"add": ea + eb, "sub": ea - eb, "mul": ea * eb}[op]
        lo, hi = _INT_RANGE[dt]
        if mode == 2:
            hi = _DEC_RANGE[dt]
            lo = -hi
        if mode != 0:
            bad = np.array([(x < lo or x > hi) for x in r], dtype=bool) & valid
            if bad.any():
                raise OverflowError_("overflow")
        mask = (1 << (dt.itemsize * 8)) - 1
        wrapped = np.array([int(x) & mask for x in r], dtype=np.uint64).astype(np.dtype(f"u{dt.itemsize}"))
        return wrapped.view(dt) if dt.kind == "i" else wrapped, valid
    if op == "cast":
        a, av = eval_expr(node[2], cols, n)
        return cast(a, av, np.dtype(node[1])), av
    raise ValueError(op)


def cast(a, valid, dt):
    """CAST of the values a (valid rows only can fail) to dtype dt with DuckDB's numeric rules
    (TryCastWithOverflowCheck, numeric_cast.hpp:27-72,187-197): an integer outside the target's range and a finite
    DOUBLE that becomes an infinite FLOAT raise OverflowError_; integers round once to FLOAT / DOUBLE; an integer
    becomes BOOLEAN as `!= 0`.  FLOAT / DOUBLE -> integer is not supported (ValueError)."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        if dt.kind != "f":
            raise ValueError(f"cast {a.dtype} -> {dt} is not supported")
        with np.errstate(over="ignore"):
            r = a.astype(dt)
        if (np.isfinite(a) & np.isinf(r) & valid).any():
            raise OverflowError_("overflow")
        return r
    if dt == np.bool_:
        return a != 0
    if dt.kind == "f":
        return a.astype(dt)  # one rounding: numpy converts 64-bit integers to float32 directly
    lo, hi = _INT_RANGE[dt]
    ints = [int(x) for x in a]
    if any(ok and not lo <= x <= hi for x, ok in zip(ints, valid)):
        raise OverflowError_("overflow")
    mask = (1 << (dt.itemsize * 8)) - 1
    wrapped = np.array([x & mask for x in ints], dtype=np.uint64).astype(np.dtype(f"u{dt.itemsize}"))
    return wrapped.view(dt)


def filter_select(pred, cols, n):
    """true_sel of ExpressionExecutor::SelectExpression: rows where pred is TRUE (NULL -> dropped)."""
    v, valid = eval_expr(pred, cols, n)
    keep = v.astype(bool) & valid
    return np.nonzero(keep)[0].astype(np.uint32), keep


# ------------------------------------------------------------------ hash aggregate
def _key_tuple_arrays(key_cols, n):
    """canonical per-row key tuples: NULL is a group of its own; -0.0 == 0.0; NaNs equal."""
    parts = []
    for values, valid in key_cols:
        v = np.asarray(values)
        if v.dtype.kind == "f":
            v = v.copy()
            v[v == 0.0] = 0.0
            bits = v.view(np.uint64 if v.dtype == np.float64 else np.uint32).astype(np.uint64)
            bits[np.isnan(v)] = np.uint64(0x7FF8000000000000)
            v = bits
        parts.append((v, np.ones(n, dtype=bool) if valid is None else valid))
    return parts


def group_by(key_cols, aggs, n):
    """GROUP BY with DuckDB semantics.
    aggs: list of (func, (values, valid) | None), func in
    count_star count sum sum_no_overflow min max avg.
    Returns dict: key tuple (None for NULL; float keys as canonical bit patterns) -> list of results.
    sum(int) -> python int (hugeint), sum(float) -> float (np.float64 sequential order not guaranteed),
    avg -> float, computed like IntegerAverageOperationHugeint (avg.cpp:109-121): long double(sum)/count.
    Reference: GroupedAggregateHashTable::AddChunk (aggregate_hashtable.cpp:630-743), sum.cpp, avg.cpp."""
    parts = _key_tuple_arrays(key_cols, n)
    groups = {}
    order = []
    keys = []
    for r in range(n):
        k = tuple((p[0][r].item() if p[1][r] else None) for p in parts)
        keys.append(k)
    for r, k in enumerate(keys):
        if k not in groups:
            groups[k] = []
            order.append(k)
        groups[k].append(r)
    out = {}
    for k in order:
        rows = np.array(groups[k], dtype=np.int64)
        res = []
        for func, col in aggs:
            if func == "count_star":
                res.append(len(rows))
                continue
            v, valid = col
            vv = np.ones(n, dtype=bool) if valid is None else valid
            sel = rows[vv[rows]]
            x = np.asarray(v)[sel]
            if func == "count":
                res.append(len(sel))
            elif len(sel) == 0:
                res.append(None)
            elif func in ("sum", "sum_no_overflow"):
                if x.dtype.kind == "f":
                    res.append(float(np.sum(x.astype(np.float64))))
                else:
                    s = int(np.sum(x.astype(object)))
                    if func == "sum_no_overflow":
                        s = (s + 2 ** 63) % 2 ** 64 - 2 ** 63
                    res.append(s)
            elif func == "avg":
                if x.dtype.kind == "f":
                    res.append(float(np.sum(x.astype(np.float64))) / len(sel))
                else:
                    s = int(np.sum(x.astype(object)))
                    res.append(float(np.longdouble(s) / np.longdouble(len(sel))))
            elif func in ("min", "max"):
                if x.dtype.kind == "f":
                    nan = np.isnan(x)
                    if func == "max":
                        res.append(float("nan") if nan.any() else float(x.max()))
                    else:
                        res.append(float("nan") if nan.all() else float(x[~nan].min()))
                else:
                    res.append(int(x.min() if func == "min" else x.max()))
            else:
                raise ValueError(func)
        out[k] = res
    return out


# ------------------------------------------------------------------ hash join
def hash_join(build_keys, probe_keys, n_build, n_probe, join_type="inner"):
    """Equality join on key columns with DuckDB semantics: NULL keys never match
    (join_hashtable.cpp:714-742); -0.0 == +0.0, NaN == NaN.
    Returns, by join type:
      inner: sorted list of (probe_row, build_row)
      left : same plus (probe_row, -1) for probe rows without a partner
      semi / anti: sorted probe rows with / without a partner
      mark : (matched bool array, valid bool array)  (ScanStructure::NextMarkJoin, join_hashtable.cpp:2001+)"""
    bparts = _key_tuple_arrays(build_keys, n_build)
    pparts = _key_tuple_arrays(probe_keys, n_probe)
    table = {}
    build_has_null = False
    for r in range(n_build):
        if not all(p[1][r] for p in bparts):
            build_has_null = True
            continue
        k = tuple(p[0][r].item() for p in bparts)
        table.setdefault(k, []).append(r)
    pairs, semi, anti = [], [], []
    matched = np.zeros(n_probe, dtype=bool)
    mvalid = np.ones(n_probe, dtype=bool)
    for r in range(n_probe):
        isnull = not all(p[1][r] for p in pparts)
        rows = [] if isnull else table.get(tuple(p[0][r].item() for p in pparts), [])
        if rows:
            matched[r] = True
            semi.append(r)
            pairs.extend((r, b) for b in rows)
        else:
            anti.append(r)
            if join_type == "left":
                pairs.append((r, -1))
            if (isnull or build_has_null) and n_build > 0:
                mvalid[r] = False
    if join_type in ("inner", "left"):
        return sorted(pairs)
    if join_type == "semi":
        return semi
    if join_type == "anti":
        return anti
    if join_type == "mark":
        return matched, mvalid
    raise ValueError(join_type)
