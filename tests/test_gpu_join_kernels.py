"""The hash-join build and generic probe (join.cu) and the radix partition (hash.cu), checked against exact references
and against the kernel trace.

Every join case gives the build side a row-id payload column and compares the whole result, as a multiset of rows,
with the oracle's (probe row, build row) pairs: lhs_sel, every lhs and payload value bit for bit, every validity bit,
the MARK value and its validity, and the returned count.  lhs_sel is a caller-owned buffer filled with a sentinel and
sized for the true result plus a margin, so a probe that writes past its count or capacity changes sentinels instead
of memory it does not own.  The inverse of murmur64 (oracle.port.murmur64_inverse) builds the collisions random data
never makes: two composite keys with one 64-bit hash, a composite hash equal to the table's empty-slot key, clusters of
keys whose home slots are the last slots of the table, and partitions chosen row by row."""
import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran
from oracle import port as P
from test_gpu_agg_kernel_paths import traced_window
from test_gpu_kernel_paths import _download_raw

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of join.cu and hash.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "join_append_kernel": ["test_composite_keys", "test_build_growth_and_late_validity"],
    "join_append_col_kernel": ["test_composite_keys", "test_build_growth_and_late_validity"],
    "join_init_slots_kernel": ["test_composite_keys", "test_wrapping_clusters"],
    "join_insert_kernel": ["test_composite_keys", "test_wrapping_clusters", "test_dense_range_limit",
                           "test_dense_duplicate_falls_back"],
    "join_minmax_kernel": ["test_dense_range_limit"],
    "join_dense_build_kernel": ["test_dense_range_limit", "test_dense_duplicate_falls_back",
                                "test_dense_inline_payloads"],
    "join_inline_kernel": ["test_hash_inline_payload"],
    "join_probe_kernel": ["test_composite_keys", "test_wrapping_clusters", "test_probe_column_shapes",
                          "test_probe_capacity"],
    "fill_u64_kernel4": ["test_probe_column_shapes"],
    "hash_kernel": ["test_hash_kernel_columns"],
    "part_hist_kernel": ["test_partition_generic", "test_partition_fast_staged"],
    "part_scatter_index_kernel": ["test_partition_generic"],
    "part_scatter_col_kernel": ["test_partition_generic"],
    "fill_u64_kernel": ["test_partition_generic"],
    "exclusive_scan_small_kernel": ["test_partition_generic", "test_partition_fast_staged"],
    "part_count_kernel": ["test_partition_fast_staged", "test_partition_fast_reg"],
    "part_move_staged_kernel": ["test_partition_fast_staged", "test_partition_fast_reg", "test_partition_scatter_peer"],
    "part_move_reg_kernel": ["test_partition_fast_reg", "test_partition_scatter_peer"],
}
# kernels of those files that no test here has to reach, with the reason
KERNEL_EXCLUDED = {}

JT = {"inner": capi.JOIN_INNER, "left": capi.JOIN_LEFT, "semi": capi.JOIN_SEMI, "anti": capi.JOIN_ANTI,
      "mark": capi.JOIN_MARK}
JOIN_TYPES = list(JT)
EMPTY_KEY = 1 << 63          # the open-addressing table's empty-slot key (and the composite side slot's hash)
SENTINEL = 0xDEADBEEF
MARGIN = 256
ALL_DTYPES = [np.bool_, np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.float32, np.int64, np.uint64,
              np.float64]


# ------------------------------------------------------------------ helpers
def cells(vals, valid):
    """values as comparable Python ints (floats by their bits, BOOL as 0 / 1), None where NULL"""
    a = np.asarray(vals)
    if a.dtype.kind == "f":
        a = a.view(np.uint64 if a.itemsize == 8 else np.uint32)
    elif a.dtype == np.bool_:
        a = a.astype(np.uint8)
    out = a.tolist()
    if valid is not None:
        for i in np.nonzero(~np.asarray(valid, dtype=bool))[0]:
            out[i] = None
    return out


def logical(vectors, n):
    return [v.logical(n) for v in vectors]


def concat(cols_per_batch):
    """[[(vals, valid) per column] per batch] -> [(vals, valid) per column] over all batches"""
    ncol = len(cols_per_batch[0])
    return [(np.concatenate([b[c][0] for b in cols_per_batch]), np.concatenate([b[c][1] for b in cols_per_batch]))
            for c in range(ncol)]


def random_values(rng, dtype, n):
    dtype = np.dtype(dtype)
    if dtype == np.bool_:
        return rng.random(n) < 0.5
    if dtype.kind == "f":
        v = rng.standard_normal(n).astype(dtype)
        v[rng.random(n) < 0.1] = np.nan
        v[rng.random(n) < 0.1] = -0.0
        return v
    info = np.iinfo(dtype)
    return rng.integers(info.min, info.max, size=n, endpoint=True, dtype=dtype)


def sel_buffer(length):
    import torch
    return torch.full((max(1, length),), SENTINEL - (1 << 32), dtype=torch.int32, device="cuda:0")


class JoinRun:
    """One join: create, sink every build batch, finalize, probe once into a sentinel-filled lhs_sel buffer."""

    def __init__(self, jt, key_types, pay_types, builds, nkeys, probe, npb, nlhs, out_capacity=0, sel_len=None):
        self.jt, self.key_types, self.pay_types, self.builds = jt, key_types, pay_types, builds
        self.nkeys, self.probe, self.npb, self.nlhs = nkeys, probe, npb, nlhs
        self.out_capacity, self.sel_len = out_capacity, sel_len

    def __call__(self, ctx):
        """-> (error code or None, count, result columns, lhs_sel words as uint32)"""
        import torch
        j = ops.HashJoin(ctx, JT[self.jt], self.key_types, self.pay_types)
        npay = len(self.pay_types)
        for batch, _ in self.builds:
            j.sink(batch, list(range(self.nkeys)), list(range(self.nkeys, self.nkeys + npay)))
        j.finalize()
        sel = sel_buffer(self.sel_len)
        code, count, res = None, None, None
        try:
            out, count = j.execute(self.probe, list(range(self.nkeys)), list(range(self.nkeys, self.nkeys + self.nlhs)),
                                   self.out_capacity, sel.data_ptr())
            res = _download_raw(out)
            out.free()
        except capi.B200Error as e:
            code = e.code
        torch.cuda.synchronize()
        words = sel.cpu().numpy().view(np.uint32).copy()
        j.close()
        return code, count, res, words


def expected_rows(jt, bkeys, bpay, pkeys, plhs, nb, npb):
    """the oracle's result as a sorted list of rows (probe row, lhs cells, payload cells | mark cell)"""
    lhs = [cells(v, ok) for v, ok in plhs]
    pay = [cells(v, ok) for v, ok in bpay]
    r = P.hash_join(bkeys, pkeys, nb, npb, jt)
    if jt in ("inner", "left"):
        rows = [(p, tuple(c[p] for c in lhs), tuple(c[b] if b >= 0 else None for c in pay)) for p, b in r]
    elif jt in ("semi", "anti"):
        rows = [(p, tuple(c[p] for c in lhs), ()) for p in r]
    else:
        matched, mvalid = r
        mark = cells(matched, mvalid)
        rows = [(p, tuple(c[p] for c in lhs), (mark[p],)) for p in range(npb)]
    return sorted(rows, key=repr)


def result_rows(jt, res, words, count, nlhs):
    got_cols = [cells(v, ok) for v, ok in res]
    rows = [(int(words[i]), tuple(c[i] for c in got_cols[:nlhs]), tuple(c[i] for c in got_cols[nlhs:]))
            for i in range(count)]
    return sorted(rows, key=repr)


def check_join(ctx, jt, key_types, pay_types, builds, nkeys, probe, probe_cols, npb, nlhs, always=("join_append_kernel",)):
    """run the join in a traced window and compare with the oracle -> kernel names.  builds: [(Batch, logical columns)]
    with key columns, then payload columns; probe_cols: the probe batch's logical columns (keys, then lhs)."""
    bcols = concat([cols for _, cols in builds]) if builds else None
    nb = len(bcols[0][0]) if bcols else 0
    if bcols is None:
        bcols = [(np.zeros(0, dtype=capi.DTYPE_OF_TYPE[t]), np.zeros(0, dtype=bool)) for t in key_types + pay_types]
    exp = expected_rows(jt, bcols[:nkeys], bcols[nkeys:] if jt in ("inner", "left") else [], probe_cols[:nkeys],
                        probe_cols[nkeys:nkeys + nlhs], nb, npb)
    run = JoinRun(jt, key_types, pay_types, builds, nkeys, probe, npb, nlhs, sel_len=len(exp) + MARGIN)
    (code, count, res, words), names = traced_window(lambda: run(ctx), [k for k in always if nb])
    assert code is None, code
    assert count == len(exp), (count, len(exp))
    assert (words[count:] == SENTINEL).all(), "lhs_sel was written past the result"
    got = result_rows(jt, res, words, count, nlhs)
    assert len(res) == nlhs + (len(pay_types) if jt in ("inner", "left") else 1 if jt == "mark" else 0)
    assert got == exp, next((g, e) for g, e in zip(got, exp) if g != e) if len(got) == len(exp) else len(got)
    return names


def upload(ctx, vectors, n):
    return ops.Batch.upload(ctx, vectors, n), logical(vectors, n)


def flat(vals, valid=None):
    return ops.Vector.flat(vals, valid)


def dictionary_of(vals, valid, rng):
    """the same logical column as a dictionary vector: a shuffled dictionary with a spare entry, and a selection"""
    n = len(vals)
    perm = rng.permutation(n + 1)
    d = np.empty(n + 1, dtype=vals.dtype)
    dv = np.ones(n + 1, dtype=bool)
    d[perm[:n]] = vals
    dv[perm[:n]] = True if valid is None else valid
    d[perm[n]] = vals[0] if n else d[perm[n]]
    return ops.Vector.dictionary(d, perm[:n].astype(np.uint32), None if valid is None else dv)


# ------------------------------------------------------------------ composite keys
def composite_data(rng, nkeys, nb, npb):
    """build / probe key columns (nkeys - 1 mixed columns, then a BIGINT column solved for the hash) with:
    duplicate build keys; pairs of different build keys with one full hash; keys hashing to EMPTY_KEY (side slot),
    duplicated, and a different probe key with the same EMPTY_KEY hash; NULLs in every position; +-0.0 and NaN"""
    types = [np.int32, np.float64, np.int16][:nkeys - 1]
    pools = {np.int32: np.array([-2 ** 31, 2 ** 31 - 1, 0, 7, -7], dtype=np.int32),
             np.float64: np.array([0.0, -0.0, np.nan, 2.5, -np.inf], dtype=np.float64),
             np.int16: np.array([-32768, 32767, 0, 1], dtype=np.int16)}

    def side(n):
        cols = [(rng.choice(pools[t], size=n), rng.random(n) > 0.06) for t in types]
        last = rng.integers(-3, 4, size=n).astype(np.int64)
        return cols, last, rng.random(n) > 0.06

    bcols, blast, blv = side(nb)
    pcols, plast, plv = side(npb)

    def prefix(cols, i):
        return int(P.hash_columns([(c[i:i + 1], v[i:i + 1]) for c, v in cols])[0])

    def full(cols, last, lv, i):
        return int(P.hash_columns([(c[i:i + 1], v[i:i + 1]) for c, v in cols] + [(last[i:i + 1], lv[i:i + 1])])[0])

    pool0 = list(pools[types[0]])

    def other(v, *avoid):
        """a value of the first key column's pool that differs from v and from every value in avoid"""
        return next(x for x in pool0 if x != v and x not in avoid)

    def solve(cols, last, i, target):
        last[i] = np.uint64(P.combine_hash_preimage(prefix(cols, i), target)).view(np.int64)

    # forced full-hash collisions: build row k + 1 gets the full hash of build row k with a different first column
    for k in range(0, 40, 2):
        for c, v in bcols:
            v[k] = v[k + 1] = True
        blv[k] = blv[k + 1] = True
        bcols[0][0][k + 1] = other(bcols[0][0][k])
        solve(bcols, blast, k + 1, full(bcols, blast, blv, k))
        for j in (k, k + 1):        # both keys are probed
            for (c, v), (pc, pv) in zip(bcols, pcols):
                pc[j], pv[j] = c[j], True
            plast[j], plv[j] = blast[j], True
    for k in range(40):             # and both are duplicated in the build
        for c, v in bcols:
            c[40 + k], v[40 + k] = c[k], v[k]
        blast[40 + k], blv[40 + k] = blast[k], blv[k]
    # composite hash == EMPTY_KEY (the side slot): rows 80 and 81 hold one key, row 82 another
    for c, v in bcols:
        v[80] = v[81] = v[82] = True
        c[81] = c[80]
    blv[80] = blv[81] = blv[82] = True
    bcols[0][0][82] = other(bcols[0][0][80])
    for i in (80, 81, 82):
        solve(bcols, blast, i, EMPTY_KEY)
    for j, src in ((50, 80), (51, 82)):
        for (c, v), (pc, pv) in zip(bcols, pcols):
            pc[j], pv[j] = c[src], True
        plast[j], plv[j] = blast[src], True
    # a probe key with the EMPTY_KEY hash that no build row holds
    for c, v in pcols:
        v[52] = True
    plv[52] = True
    pcols[0][0][52] = other(bcols[0][0][80], bcols[0][0][82])
    solve(pcols, plast, 52, EMPTY_KEY)
    bk = bcols + [(blast, blv)]
    pk = pcols + [(plast, plv)]
    bh, ph = P.hash_columns(bk), P.hash_columns(pk)
    assert bh[1] == bh[0] and (bh == np.uint64(EMPTY_KEY)).sum() == 3 and ph[52] == np.uint64(EMPTY_KEY)
    return bk, pk


@pytest.mark.parametrize("nkeys", [2, 4])
@pytest.mark.parametrize("jt", JOIN_TYPES)
def test_composite_keys(ctx, jt, nkeys):
    """2 and 4 key columns, every join type: chains that hold two different keys with one 64-bit hash (probe_first /
    chain_next must compare the stored key columns), the side slot for a hash equal to EMPTY_KEY with duplicates in
    it, NULLs in every key position on both sides (MARK: NULL where the build side holds a NULL key)"""
    rng = np.random.default_rng(100 + nkeys * 10 + JOIN_TYPES.index(jt))
    nb, npb = 300, 400
    bk, pk = composite_data(rng, nkeys, nb, npb)
    rid = np.arange(nb, dtype=np.int64)
    lhs = [(random_values(rng, np.int32, npb), rng.random(npb) > 0.2), (random_values(rng, np.float64, npb), None)]
    bt = [capi.TYPE_OF_DTYPE[np.asarray(v).dtype] for v, _ in bk]
    builds = [upload(ctx, [flat(v[:120], ok[:120]) for v, ok in bk] + [flat(rid[:120])], 120),
              upload(ctx, [flat(v[120:], ok[120:]) for v, ok in bk] + [flat(rid[120:])], nb - 120)]
    pb, pcols = upload(ctx, [flat(v, ok) for v, ok in pk] + [flat(v, ok) for v, ok in lhs], npb)
    names = check_join(ctx, jt, bt, [capi.INT64], builds, nkeys, pb, pcols, npb, 2)
    assert_ran(names, "join_append_kernel", "join_append_col_kernel", "join_init_slots_kernel", "join_insert_kernel",
               "join_probe_kernel<1>")
    assert_not_ran(names, "join_probe_tile_kernel", "join_dense_build_kernel", "join_inline_kernel")
    if jt in ("inner", "left"):
        assert_ran(names, "join_probe_kernel<0>")       # composite keys are never unique: the counting pass sizes it
    else:
        assert_not_ran(names, "join_probe_kernel<0>")   # at most one row per probe row


# ------------------------------------------------------------------ wrapping clusters
def table_cap(rows, load):
    cap = 1024
    while cap * load < rows:
        cap <<= 1
    return cap


def keys_with_slots(rng, slots, cap):
    """64-bit keys whose home slot murmur64(key) & (cap - 1) is the given one"""
    shift = cap.bit_length() - 1
    out = []
    for s in slots:
        while True:
            h = ((int(rng.integers(0, 2 ** 62)) << shift) | int(s)) & ((1 << 64) - 1)
            k = P.murmur64_inverse(h)
            if k != EMPTY_KEY:
                out.append(k)
                break
    return np.array(out, dtype=np.uint64)


@pytest.mark.parametrize("load", ["0.5", "0.9"])
@pytest.mark.parametrize("probe_kind", ["flat", "dict"])
@pytest.mark.parametrize("dtype", [np.int64, np.uint64])
def test_wrapping_clusters(ctx, monkeypatch, dtype, probe_kind, load):
    """single BIGINT / UBIGINT keys whose home slots are the last 6 slots of the table: the cluster wraps from the last
    slot to slot 0, where other keys live too; duplicates chain; EMPTY_KEY (INT64_MIN / 2^63) goes to the side slot.
    Absent probe keys that land inside the cluster walk it and stop at the first empty slot.  Flat nullable probe keys
    take the tile kernel, a dictionary probe key the generic one."""
    monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    monkeypatch.setenv("B200_JOIN_LOAD", load)
    rng = np.random.default_rng(7 + (dtype == np.uint64) * 2 + (probe_kind == "dict") * 4 + (load == "0.9") * 8)
    nb = 600
    cap = table_cap(nb, float(load))
    tail = keys_with_slots(rng, [cap - 1 - (i % 6) for i in range(60)], cap)
    head = keys_with_slots(rng, [i % 8 for i in range(30)], cap)
    rest = keys_with_slots(rng, rng.integers(0, cap, size=nb - 60 - 30 - 30 - 4), cap)
    uniq = np.concatenate([tail, head, rest, np.array([EMPTY_KEY], dtype=np.uint64)])
    bk = np.concatenate([uniq, tail[:30], np.array([EMPTY_KEY] * 3, dtype=np.uint64)])
    assert len(bk) == nb
    perm = rng.permutation(nb)
    bk = bk[perm].view(dtype)
    absent = keys_with_slots(rng, [cap - 1 - (i % 6) for i in range(40)] + [i % 8 for i in range(40)], cap)
    npb = 3000
    pk = np.concatenate([uniq[rng.integers(0, len(uniq), size=npb - 200)], absent,
                         np.array([EMPTY_KEY] * 20, dtype=np.uint64), rng.integers(0, 2 ** 64, size=100, dtype=np.uint64)])
    pk = pk[rng.permutation(npb)].view(dtype)
    pkv = rng.random(npb) > 0.05
    lhs = random_values(rng, np.int64, npb)
    rid = np.arange(nb, dtype=np.int64)
    builds = [upload(ctx, [flat(bk), flat(rid)], nb)]
    key_vec = flat(pk, pkv) if probe_kind == "flat" else dictionary_of(pk, pkv, rng)
    pb, pcols = upload(ctx, [key_vec, flat(lhs)], npb)
    tk = capi.TYPE_OF_DTYPE[np.dtype(dtype)]
    for jt in ("inner", "semi", "mark"):
        names = check_join(ctx, jt, [tk], [capi.INT64], builds, 1, pb, pcols, npb, 1)
        assert_ran(names, "join_init_slots_kernel", "join_insert_kernel")
        assert_not_ran(names, "join_dense_build_kernel")
        if probe_kind == "flat":
            assert_ran(names, "join_probe_tile_kernel<false, false>")
            assert_not_ran(names, "join_probe_kernel<1>")
        else:
            assert_ran(names, "join_probe_kernel<1>")
            assert_not_ran(names, "join_probe_tile_kernel")


# ------------------------------------------------------------------ probe column shapes
def unaligned_batch(ctx, cols):
    """flat device columns whose data pointers sit 8 bytes past a 16-byte boundary (Batch.wrap)"""
    import torch
    keep, spec = [], []
    for vals, valid in cols:
        raw = np.ascontiguousarray(vals).view(np.uint8)
        t = torch.zeros(len(raw) + 64, dtype=torch.uint8, device="cuda:0")
        t[8:8 + len(raw)] = torch.from_numpy(raw.copy()).to("cuda:0")
        keep.append(t)
        entry = [t.data_ptr() + 8, capi.TYPE_OF_DTYPE[np.asarray(vals).dtype]]
        if valid is not None:
            w = torch.from_numpy(capi.validity_words(valid).view(np.int64).copy()).to("cuda:0")
            keep.append(w)
            entry.append(w.data_ptr())
        spec.append(tuple(entry))
    assert all((s[0] & 15) == 8 for s in spec)
    return ops.Batch.wrap(ctx, spec, len(cols[0][0]), keepalive=keep)


@pytest.mark.parametrize("shape", ["dict", "const", "null_const", "unaligned"])
def test_probe_column_shapes(ctx, shape):
    """the generic probe's column loads: a dictionary, constant, NULL constant or unaligned probe key and lhs columns
    of every width with validity (also as dictionaries and constants), through INNER, LEFT and MARK"""
    rng = np.random.default_rng(["dict", "const", "null_const", "unaligned"].index(shape) + 300)
    nb, npb = 400, 2000
    bk = rng.integers(-20, 20, size=nb).astype(np.int32)
    bkv = rng.random(nb) > 0.05
    rid = np.arange(nb, dtype=np.int64)
    builds = [upload(ctx, [flat(bk, bkv), flat(rid)], nb)]
    pk = rng.integers(-25, 25, size=npb).astype(np.int32)
    pkv = rng.random(npb) > 0.1
    lhs = [(random_values(rng, dt, npb), rng.random(npb) > 0.15) for dt in ALL_DTYPES]
    if shape == "unaligned":
        pb = unaligned_batch(ctx, [(pk, pkv)] + lhs)
        pcols = [(pk, pkv)] + lhs
    else:
        if shape == "dict":
            kv = dictionary_of(pk, pkv, rng)
        elif shape == "const":
            kv = ops.Vector.constant(int(bk[np.nonzero(bkv)[0][0]]), np.int32)
        else:
            kv = ops.Vector.constant(0, np.int32, is_null=True)
        lv = [dictionary_of(v, ok, rng) if i % 3 == 0 else flat(v, ok) if i % 3 == 1 else
              ops.Vector.constant(v[0].item(), v.dtype, is_null=not ok[0]) for i, (v, ok) in enumerate(lhs)]
        pb, pcols = upload(ctx, [kv] + lv, npb)
    for jt in ("inner", "left", "mark"):
        names = check_join(ctx, jt, [capi.INT32], [capi.INT64], builds, 1, pb, pcols, npb, len(lhs))
        assert_ran(names, "join_probe_kernel<1>")
        assert_not_ran(names, "join_probe_tile_kernel")
        if jt != "inner":       # one result row per probe row: the nullable output columns are initialised
            assert_ran(names, "fill_u64_kernel4")


def test_lhs_and_payload_limits(ctx):
    """12 lhs columns and 12 payload columns (one of them the row id) pass through exactly; 13 of either is rejected"""
    rng = np.random.default_rng(12)
    nb, npb = 500, 1500
    bk = rng.integers(0, 300, size=nb).astype(np.int64)
    pays = [(random_values(rng, ALL_DTYPES[i % 11], nb), rng.random(nb) > 0.1 if i % 2 else None) for i in range(11)]
    pays.append((np.arange(nb, dtype=np.int64), None))
    pt = [capi.TYPE_OF_DTYPE[v.dtype] for v, _ in pays]
    builds = [upload(ctx, [flat(bk)] + [flat(v, ok) for v, ok in pays], nb)]
    pk = rng.integers(0, 350, size=npb).astype(np.int64)
    lhs = [(random_values(rng, ALL_DTYPES[(i + 5) % 11], npb), rng.random(npb) > 0.1) for i in range(12)]
    pb, pcols = upload(ctx, [flat(pk)] + [flat(v, ok) for v, ok in lhs], npb)
    for jt in ("inner", "left"):
        check_join(ctx, jt, [capi.INT64], pt, builds, 1, pb, pcols, npb, 12)
    with pytest.raises(capi.B200Error) as e:
        ops.HashJoin(ctx, capi.JOIN_INNER, [capi.INT64], pt + [capi.INT32])
    assert e.value.code == capi.ERR_INVALID
    j = ops.HashJoin(ctx, capi.JOIN_INNER, [capi.INT64], pt)
    j.sink(builds[0][0], [0], list(range(1, 13)))
    j.finalize()
    pb13 = ops.Batch.upload(ctx, [flat(pk)] + [flat(v, ok) for v, ok in lhs] + [flat(pk)], npb)
    with pytest.raises(capi.B200Error) as e:
        j.execute(pb13, [0], list(range(1, 14)))
    assert e.value.code == capi.ERR_INVALID
    j.close()


# ------------------------------------------------------------------ build side
def test_build_growth_and_late_validity(ctx):
    """five sink batches (one empty) grow the store 1024 -> 2048 -> 4096 -> 16384 rows.  Payload A gets its first NULL
    in batch 2 and the store regrows in batch 3: A's batch-2 NULLs must survive the copy.  Payload B gets its first
    NULL in batch 3, after a regrow.  Dictionary and constant key and payload columns in some batches."""
    rng = np.random.default_rng(55)
    sizes = [700, 900, 0, 2600, 9000]
    builds = []
    base = 0
    for i, n in enumerate(sizes):
        k = rng.integers(0, 5000, size=n).astype(np.int64)
        kv = rng.random(n) > 0.03
        a = random_values(rng, np.int32, n)
        b = random_values(rng, np.int16, n)
        rid = np.arange(base, base + n, dtype=np.int64)
        base += n
        av = (rng.random(n) > 0.2) if i >= 1 else None
        bv = (rng.random(n) > 0.2) if i >= 3 else None
        if i == 1:
            kvec = dictionary_of(k, kv, rng)
            avec = flat(a, av)
            bvec = ops.Vector.constant(int(b[0]) if n else 0, np.int16)
        elif i == 3:
            kvec = ops.Vector.constant(77, np.int64)
            avec = dictionary_of(a, av, rng)
            bvec = flat(b, bv)
        else:
            kvec, avec, bvec = flat(k, kv), flat(a, av), flat(b, bv)
        builds.append(upload(ctx, [kvec, avec, bvec, flat(rid)], n))
    nb = base
    npb = 6000
    pk = rng.integers(0, 5200, size=npb).astype(np.int64)
    pk[:50] = 77
    pb, pcols = upload(ctx, [flat(pk), flat(np.arange(npb, dtype=np.int32))], npb)
    for jt in ("inner", "left"):
        names = check_join(ctx, jt, [capi.INT64], [capi.INT32, capi.INT16, capi.INT64], builds, 1, pb, pcols, npb, 1)
        assert_ran(names, "join_append_kernel", "join_append_col_kernel", "join_insert_kernel")
    assert nb > 8192


# ------------------------------------------------------------------ dense table
DENSE_CASES = {"i64_min": (np.int64, -2 ** 63), "u64_max": (np.uint64, 2 ** 64 - 2 ** 20), "i32": (np.int32, -5000)}


def dense_keys(rng, dtype, lo, nb, span):
    """nb unique keys in [lo, lo + span) that include both ends"""
    off = np.concatenate([[0, span - 1], rng.choice(np.arange(1, span - 1), size=nb - 2, replace=False)])
    return (np.array([lo + int(o) for o in off], dtype=object).astype(np.uint64 if dtype == np.uint64 else np.int64)
            .astype(dtype))


@pytest.mark.parametrize("case", list(DENSE_CASES))
def test_dense_range_limit(ctx, case):
    """a key range of exactly max(8 x rows, 2^20) builds the dense table (join_dense_build_kernel, no
    join_insert_kernel); one more key value of range builds the hash table.  Keys near INT64_MIN / 2^64 - 1; probe keys
    far outside the range make key - dense_min wrap."""
    dtype, lo = DENSE_CASES[case]
    rng = np.random.default_rng(list(DENSE_CASES).index(case) + 400)
    nb = 1000
    limit = max(8 * nb, 1 << 20)
    tk = capi.TYPE_OF_DTYPE[np.dtype(dtype)]
    info = np.iinfo(dtype)
    for span, dense in ((limit, True), (limit + 1, False)):
        bk = dense_keys(rng, dtype, min(lo, int(info.max) - span + 1), nb, span)
        rid = np.arange(nb, dtype=np.int64)
        builds = [upload(ctx, [flat(bk), flat(rid)], nb)]
        far = np.array([info.max, info.min, info.max // 2, info.min // 2 if info.min else 1, 0, 1], dtype=dtype)
        pk = np.concatenate([bk[rng.integers(0, nb, size=1500)], far, (bk[:200].astype(np.uint64) + np.uint64(1))
                             .astype(dtype)])
        npb = len(pk)
        pb, pcols = upload(ctx, [flat(pk), flat(np.arange(npb, dtype=np.int64))], npb)
        for jt in ("inner", "anti"):
            names = check_join(ctx, jt, [tk], [capi.INT64], builds, 1, pb, pcols, npb, 1)
            assert_ran(names, "join_minmax_kernel")
            if dense:
                assert_ran(names, "join_dense_build_kernel")
                assert_not_ran(names, "join_insert_kernel", "join_init_slots_kernel")
            else:
                assert_ran(names, "join_insert_kernel")
                assert_not_ran(names, "join_dense_build_kernel")


def test_dense_duplicate_falls_back(ctx):
    """unique keys in a small range plus one duplicate: the dense build sees it and the hash table takes over, with
    the duplicate's chain"""
    rng = np.random.default_rng(8)
    nb = 2000
    bk = rng.permutation(5000)[:nb].astype(np.int64)
    bk[-1] = bk[17]
    rid = np.arange(nb, dtype=np.int64)
    builds = [upload(ctx, [flat(bk), flat(rid)], nb)]
    pk = rng.integers(-10, 5010, size=4000).astype(np.int64)
    pk[:30] = bk[17]
    pb, pcols = upload(ctx, [flat(pk), flat(pk)], 4000)
    for jt in ("inner", "left", "semi"):
        names = check_join(ctx, jt, [capi.INT64], [capi.INT64], builds, 1, pb, pcols, 4000, 1)
        assert_ran(names, "join_dense_build_kernel", "join_insert_kernel")


INLINE_DENSE = {"i8": [np.int8], "i16": [np.int16], "i8_i8": [np.int8, np.int8], "i8_i16": [np.int8, np.int16],
                "i16_u8": [np.int16, np.uint8]}


@pytest.mark.parametrize("probe_kind", ["flat", "dict"])
@pytest.mark.parametrize("pays", list(INLINE_DENSE))
def test_dense_inline_payloads(ctx, pays, probe_kind):
    """1-3 bytes of payload in one or two columns, negative INT8 / INT16 values, packed into the dense entry and
    unpacked by the tile kernel (flat probe) and by the generic probe (dictionary probe key)"""
    rng = np.random.default_rng(list(INLINE_DENSE).index(pays) * 2 + (probe_kind == "dict") + 500)
    nb = 3000
    bk = rng.permutation(10000)[:nb].astype(np.int64) - 5000
    bkv = np.ones(nb, dtype=bool)
    bkv[:20] = False
    cols = [random_values(rng, dt, nb) for dt in INLINE_DENSE[pays]]
    for c in cols:
        c[:100] = np.iinfo(c.dtype).min
        c[100:200] = -1 if c.dtype.kind == "i" else np.iinfo(c.dtype).max
    pt = [capi.TYPE_OF_DTYPE[c.dtype] for c in cols]
    builds = [upload(ctx, [flat(bk, bkv)] + [flat(c) for c in cols], nb)]
    npb = 8000
    pk = rng.integers(-5100, 5100, size=npb).astype(np.int64)
    pk[:300] = bk[rng.integers(0, 300, size=300)]
    kvec = flat(pk) if probe_kind == "flat" else dictionary_of(pk, None, rng)
    pb, pcols = upload(ctx, [kvec, flat(np.arange(npb, dtype=np.int64))], npb)
    # no row-id payload here: the inline shape allows at most 3 bytes; payload values identify the build row instead
    for jt in ("inner", "left", "mark"):
        names = check_join(ctx, jt, [capi.INT64], pt, builds, 1, pb, pcols, npb, 1)
        assert_ran(names, "join_dense_build_kernel")
        assert_not_ran(names, "join_insert_kernel")
        # a flat probe takes a tile kernel (the lean one for INNER), a dictionary key the generic probe
        (assert_ran if probe_kind == "dict" else assert_not_ran)(names, "join_probe_kernel<1>")


INLINE_HASH = {"i32": ([np.int32], True), "f32": ([np.float32], True), "i16_i16": ([np.int16, np.int16], True),
               "i8_i16_i8": ([np.int8, np.int16, np.int8], True), "i32_i8": ([np.int32, np.int8], False),
               "i32_nullable": ([np.int32], False)}


@pytest.mark.parametrize("pays", list(INLINE_HASH))
def test_hash_inline_payload(ctx, monkeypatch, pays):
    """unique keys on the hash table: a payload of exactly 4 bytes (INT32, FLOAT, two INT16s, INT8 + INT16 + INT8) is
    copied into the slot by join_inline_kernel; 5 bytes or a nullable payload are not"""
    monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    dts, inline = INLINE_HASH[pays]
    rng = np.random.default_rng(list(INLINE_HASH).index(pays) + 600)
    nb = 3000
    bk = np.unique(rng.integers(-2 ** 63, 2 ** 63, size=nb, dtype=np.int64))
    nb = len(bk)
    cols = [random_values(rng, dt, nb) for dt in dts]
    for c in cols:
        if c.dtype.kind == "i":
            c[:50] = np.iinfo(c.dtype).min
            c[50:100] = -1
    valid = (rng.random(nb) > 0.1) if pays == "i32_nullable" else None
    pt = [capi.TYPE_OF_DTYPE[c.dtype] for c in cols]
    builds = [upload(ctx, [flat(bk)] + [flat(c, valid) for c in cols], nb)]
    npb = 6000
    pk = np.concatenate([bk[rng.integers(0, nb, size=npb - 1000)], rng.integers(-2 ** 63, 2 ** 63, size=1000,
                                                                                 dtype=np.int64)])
    for probe_kind in ("flat", "dict"):
        kvec = flat(pk) if probe_kind == "flat" else dictionary_of(pk, None, rng)
        pb, pcols = upload(ctx, [kvec, flat(np.arange(npb, dtype=np.int64))], npb)
        for jt in ("inner", "left"):
            names = check_join(ctx, jt, [capi.INT64], pt, builds, 1, pb, pcols, npb, 1)
            assert_ran(names, "join_insert_kernel")
            (assert_ran if inline else assert_not_ran)(names, "join_inline_kernel")


def test_mark_null_build_keys(ctx, monkeypatch):
    """`k IN (SELECT k FROM b)`: a build side of only NULL keys, an empty one, and one with a NULL among other keys, on
    the dense table and on the hash table"""
    rng = np.random.default_rng(77)
    npb = 300
    pk = rng.integers(0, 10, size=npb).astype(np.int64)
    pkv = rng.random(npb) > 0.2
    pb, pcols = upload(ctx, [flat(pk, pkv), flat(np.arange(npb, dtype=np.int32))], npb)
    cases = {"nulls": (np.arange(5, dtype=np.int64), np.zeros(5, dtype=bool)),
             "empty": (np.zeros(0, dtype=np.int64), np.zeros(0, dtype=bool)),
             "mixed": (np.array([1, 3, 5, 0, 7], dtype=np.int64), np.array([True, True, True, False, True]))}
    for no_dense in (False, True):
        if no_dense:
            monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
        for name, (k, kv) in cases.items():
            builds = [upload(ctx, [flat(k, kv)], len(k))] if len(k) else []
            names = check_join(ctx, "mark", [capi.INT64], [], builds, 1, pb, pcols, npb, 1)
            if name == "mixed":
                assert_ran(names, "join_insert_kernel" if no_dense else "join_dense_build_kernel")


# ------------------------------------------------------------------ capacity
@pytest.mark.parametrize("probe_kind", ["flat", "dict"])
def test_probe_capacity(ctx, probe_kind):
    """out_capacity equal to the true count succeeds; one less, and the probe batch's row count for a join with
    duplicates (what the DuckDB binding tries first), return B200_ERR_CAPACITY.  No lhs_sel word at or past the
    capacity changes (the buffer holds the full result plus a margin)."""
    import torch
    rng = np.random.default_rng(900 + (probe_kind == "dict"))
    nb, npb = 3000, 5000
    bk = rng.integers(0, 1000, size=nb).astype(np.int64)
    builds = [upload(ctx, [flat(bk), flat(np.arange(nb, dtype=np.int64))], nb)]
    pk = rng.integers(0, 1100, size=npb).astype(np.int64)
    kvec = flat(pk) if probe_kind == "flat" else dictionary_of(pk, None, rng)
    pb, pcols = upload(ctx, [kvec, flat(np.arange(npb, dtype=np.int64))], npb)
    bcols = builds[0][1]
    exp = expected_rows("inner", bcols[:1], bcols[1:], pcols[:1], pcols[1:], nb, npb)
    true = len(exp)
    assert true > npb
    for cap, ok in ((true, True), (true - 1, False), (npb, False)):
        run = JoinRun("inner", [capi.INT64], [capi.INT64], builds, 1, pb, npb, 1, out_capacity=cap,
                      sel_len=true + MARGIN)
        (code, count, res, words), names = traced_window(lambda: run(ctx), ["join_append_kernel"])
        assert (words[cap:] == SENTINEL).all(), (cap, "lhs_sel written at or past the capacity")
        assert_not_ran(names, "join_probe_kernel<0>")   # a caller-given capacity: no counting pass
        if probe_kind == "dict":
            assert_ran(names, "join_probe_kernel<1>")
        else:
            assert_ran(names, "join_probe_tile_kernel")
            assert_not_ran(names, "join_probe_kernel<1>")
        if ok:
            assert code is None and count == true
            assert result_rows("inner", res, words, count, 1) == exp
        else:
            assert code == capi.ERR_CAPACITY, code
    torch.cuda.synchronize()


def int128_column(n, rng):
    import torch
    words = rng.integers(-2 ** 63, 2 ** 63, size=2 * n, dtype=np.int64)
    return torch.from_numpy(words).to("cuda:0")


def test_int128_lhs_rejected(ctx):
    """the probe copies lhs values of at most 8 bytes: an INT128 lhs column is rejected, on the tile-eligible shape
    and on the generic one"""
    import torch
    rng = np.random.default_rng(128)
    n = 1000
    bk = np.arange(n, dtype=np.int64)
    j = ops.HashJoin(ctx, capi.JOIN_INNER, [capi.INT64], [])
    j.sink(ops.Batch.upload(ctx, [flat(bk)], n), [0], [])
    j.finalize()
    key = torch.from_numpy(bk.copy()).to("cuda:0")
    big = int128_column(n, rng)
    flat_b = ops.Batch.wrap(ctx, [(key.data_ptr(), capi.INT64), (big.data_ptr(), capi.INT128)], n, keepalive=[key, big])
    sel = torch.from_numpy(np.arange(n, dtype=np.uint32).view(np.int32)).to("cuda:0")
    dict_b = ops.Batch.wrap(ctx, [(key.data_ptr(), capi.INT64, None, sel.data_ptr(), n),
                                  (big.data_ptr(), capi.INT128)], n, keepalive=[key, big, sel])
    for b in (flat_b, dict_b):
        with pytest.raises(capi.B200Error) as e:
            j.execute(b, [0], [1])
        assert e.value.code == capi.ERR_INVALID
    j.close()


# ------------------------------------------------------------------ hash.cu
def test_hash_kernel_columns(ctx):
    """b200_hash over 1-8 key columns of mixed types and vector kinds (flat with NULLs, dictionary, constant, NULL
    constant) against hash_columns"""
    import torch
    rng = np.random.default_rng(31)
    n = 5000
    vecs, cols = [], []
    for i in range(8):
        dt = ALL_DTYPES[(i * 3) % 11]
        v = random_values(rng, dt, n)
        ok = rng.random(n) > 0.1
        kind = i % 4
        vec = flat(v, ok) if kind == 0 else dictionary_of(v, ok, rng) if kind == 1 else \
            ops.Vector.constant(v[0].item(), v.dtype) if kind == 2 else ops.Vector.constant(v[0].item(), v.dtype, True)
        vecs.append(vec)
        cols.append(vec.logical(n))
    b = ops.Batch.upload(ctx, vecs, n)
    outs = [torch.zeros(n, dtype=torch.int64, device="cuda:0") for _ in range(8)]

    def run():
        # all eight in one window: a window around one small kernel is the kind the profiler most often comes back
        # from empty
        for k in range(1, 9):
            ops.hash_keys(ctx, b, list(range(k)), outs[k - 1].data_ptr())
        torch.cuda.synchronize()
        return [o.cpu().numpy().view(np.uint64).copy() for o in outs]
    got, names = traced_window(run, ["hash_kernel"])
    assert_ran(names, "hash_kernel")
    for k in range(1, 9):
        np.testing.assert_array_equal(got[k - 1], P.hash_columns(cols[:k]), err_msg=f"{k} key columns")


def check_partition(out, counts, cols, keys, bits, rid_col):
    """counts and contents of a radix partition: the row with row id r must carry row r's values and validity, and lie
    in the partition of row r's key hash"""
    n = len(cols[0][0])
    ids = P.radix_partition_ids(P.hash_columns(keys), bits) if n else np.zeros(0, dtype=np.uint32)
    np.testing.assert_array_equal(counts, np.bincount(ids, minlength=1 << bits).astype(np.uint64))
    res = _download_raw(out)
    assert len(res) == len(cols)
    rid = res[rid_col][0].astype(np.int64)
    np.testing.assert_array_equal(np.sort(rid), np.arange(n))
    off = np.concatenate([[0], np.cumsum(counts.astype(np.int64))])
    for p in range(1 << bits):
        np.testing.assert_array_equal(ids[rid[off[p]:off[p + 1]]], p)
    for c, ((gv, gok), (v, ok)) in enumerate(zip(res, cols)):
        ev = np.asarray(v)[rid]
        eok = np.ones(n, dtype=bool) if ok is None else np.asarray(ok)[rid]
        np.testing.assert_array_equal(gok, eok, err_msg=f"column {c} validity")
        view = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[ev.dtype.itemsize]
        np.testing.assert_array_equal(np.asarray(gv).view(view)[eok], ev.view(view)[eok], err_msg=f"column {c}")


def generic_columns(rng, n):
    """row id, then every width as flat-with-NULLs, a dictionary, a constant and a NULL constant"""
    vecs = [flat(np.arange(n, dtype=np.int64))]
    for i, dt in enumerate(ALL_DTYPES):
        v = random_values(rng, dt, n)
        ok = rng.random(n) > 0.1
        vecs.append(flat(v, ok) if i % 2 == 0 else dictionary_of(v, ok, rng))
    vecs.append(ops.Vector.constant(-5, np.int16))
    vecs.append(ops.Vector.constant(0, np.float64, is_null=True))
    return vecs


@pytest.mark.parametrize("bits,generic_env", [(0, True), (3, True), (5, False), (9, False), (12, False)])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 20000])
def test_partition_generic(ctx, monkeypatch, bits, generic_env, n):
    """the generic partition (part_hist -> exclusive scan -> scatter index -> one scatter per column) over nullable,
    dictionary and constant columns of every width, keyed on one column and on three"""
    if generic_env:
        monkeypatch.setenv("B200_PART_GENERIC", "1")
    rng = np.random.default_rng(bits * 1000 + n)
    vecs = generic_columns(rng, n)
    b = ops.Batch.upload(ctx, vecs, n)
    cols = logical(vecs, n)
    for key_cols in ([9], [6, 2, 12]):
        (out, counts), names = traced_window(lambda: ops.radix_partition(ctx, b, key_cols, bits),
                                             ["exclusive_scan_small_kernel"])
        check_partition(out, counts, cols, [cols[k] for k in key_cols], bits, 0)
        assert_ran(names, "exclusive_scan_small_kernel")
        if n:
            assert_ran(names, "part_hist_kernel", "part_scatter_index_kernel", "part_scatter_col_kernel",
                       "fill_u64_kernel")
        assert_not_ran(names, "part_count_kernel", "part_move_staged_kernel", "part_move_reg_kernel")


def test_partition_generic_large(ctx):
    """3 M rows through the generic path at 12 bits, key columns with NULLs"""
    rng = np.random.default_rng(3)
    n = 3_000_000
    k = rng.integers(-10 ** 6, 10 ** 6, size=n).astype(np.int32)
    kv = rng.random(n) > 0.01
    vecs = [flat(np.arange(n, dtype=np.int64)), flat(k, kv), flat(random_values(rng, np.float64, n))]
    b = ops.Batch.upload(ctx, vecs, n)
    out, counts = ops.radix_partition(ctx, b, [1, 2], 12)
    check_partition(out, counts, logical(vecs, n), logical(vecs, n)[1:], 12, 0)


def fast_columns(rng, n, key_dtype, row_bytes):
    """key, row id, then columns of 1, 2, 4 and 8 bytes padded up to row_bytes (at most 16 columns), no NULLs"""
    dts = [key_dtype, np.int64, np.uint8, np.int16, np.float32, np.float64, np.bool_, np.uint16, np.int8, np.uint32]
    total = sum(np.dtype(d).itemsize for d in dts)
    for d in (np.int64, np.int32, np.int16, np.uint8):
        while total + np.dtype(d).itemsize <= row_bytes:
            dts.append(d)
            total += np.dtype(d).itemsize
    assert total == row_bytes and len(dts) <= 16
    vals = [random_values(rng, d, n) for d in dts]
    vals[1] = np.arange(n, dtype=np.int64)
    return [flat(v) for v in vals]


@pytest.mark.parametrize("key_dtype", [np.int64, np.int32])
@pytest.mark.parametrize("row_bytes", [48, 49])
def test_partition_fast_staged(ctx, key_dtype, row_bytes):
    """the staged fast path with columns of 1, 2, 4 and 8 bytes up to the 48-byte row limit (part_count_kernel and
    part_move_staged_kernel, FAST64 for a BIGINT key); one byte more takes the generic path"""
    rng = np.random.default_rng(row_bytes + (key_dtype == np.int64))
    n = 300_007
    vecs = fast_columns(rng, n, key_dtype, row_bytes)
    b = ops.Batch.upload(ctx, vecs, n)
    cols = logical(vecs, n)
    fast64 = "true" if key_dtype == np.int64 else "false"
    for bits in (1, 4):
        (out, counts), names = traced_window(lambda: ops.radix_partition(ctx, b, [0], bits),
                                             ["exclusive_scan_small_kernel"])
        check_partition(out, counts, cols, cols[:1], bits, 1)
        if row_bytes == 48:
            assert_ran(names, f"part_count_kernel<{fast64}>", f"part_move_staged_kernel<false, {fast64}>")
            assert_not_ran(names, "part_hist_kernel", "part_move_reg_kernel")
        else:
            assert_ran(names, "part_hist_kernel")
            assert_not_ran(names, "part_count_kernel", "part_move_staged_kernel")


@pytest.mark.parametrize("bulk", ["0", "1"])
@pytest.mark.parametrize("nc", [1, 2, 3, 4])
def test_partition_fast_reg(ctx, monkeypatch, nc, bulk):
    """NC 8-byte columns with the BIGINT key among them take part_move_reg_kernel<false, NC, BULK>;
    B200_PART_NO_REG=1 sends the same shape to the staged kernel"""
    monkeypatch.setenv("B200_PART_BULK", bulk)
    rng = np.random.default_rng(nc * 2 + int(bulk))
    n = 200_003
    k = rng.integers(-2 ** 63, 2 ** 63, size=n, dtype=np.int64)
    vals = [np.arange(n, dtype=np.int64), k] + [random_values(rng, np.float64, n), random_values(rng, np.uint64, n)]
    vals = vals[:nc] if nc > 1 else [k]
    key_col = 1 if nc > 1 else 0
    vecs = [flat(v) for v in vals]
    b = ops.Batch.upload(ctx, vecs, n)
    cols = logical(vecs, n)
    for no_reg in (False, True):
        if no_reg:
            monkeypatch.setenv("B200_PART_NO_REG", "1")
        (out, counts), names = traced_window(lambda: ops.radix_partition(ctx, b, [key_col], 3),
                                             ["exclusive_scan_small_kernel"])
        if nc > 1:
            check_partition(out, counts, cols, cols[key_col:key_col + 1], 3, 0)
        else:
            ids = P.radix_partition_ids(P.hash_columns([(k, None)]), 3)
            np.testing.assert_array_equal(counts, np.bincount(ids, minlength=8).astype(np.uint64))
            got = out.download(0)[0]
            off = np.concatenate([[0], np.cumsum(counts.astype(np.int64))])
            for p in range(8):
                np.testing.assert_array_equal(np.sort(got[off[p]:off[p + 1]]), np.sort(k[ids == p]))
        assert_ran(names, "part_count_kernel<true>")
        if no_reg:
            assert_ran(names, "part_move_staged_kernel<false, true>")
            assert_not_ran(names, "part_move_reg_kernel")
        else:
            assert_ran(names, f"part_move_reg_kernel<false, {nc}, {'true' if bulk == '1' else 'false'}>")
            assert_not_ran(names, "part_move_staged_kernel")


def keys_in_partitions(rng, parts, bits):
    """BIGINT keys whose radix partition is the given one (the hash built first, the key by murmur64_inverse)"""
    sh = 48 - bits
    h = rng.integers(0, 2 ** 64, size=len(parts), dtype=np.uint64)
    h = (h & ~np.uint64(((1 << bits) - 1) << sh)) | (np.asarray(parts, dtype=np.uint64) << np.uint64(sh))
    return np.array([P.murmur64_inverse(int(x)) for x in h], dtype=np.uint64).view(np.int64)


@pytest.mark.parametrize("skew", ["one_partition", "one_empty"])
@pytest.mark.parametrize("bits", [2, 4, 9])
def test_partition_skew(ctx, skew, bits):
    """every row in one partition, and every partition but one filled, on the fast and the generic path"""
    rng = np.random.default_rng(bits * 2 + (skew == "one_empty"))
    n = 100_000 if bits <= 4 else 20_000
    nparts = 1 << bits
    if skew == "one_partition":
        parts = np.full(n, nparts - 1)
    else:
        parts = rng.integers(0, nparts - 1, size=n)
        parts[parts >= 1] += 1       # partition 1 stays empty
    k = keys_in_partitions(rng, parts, bits)
    vecs = [flat(np.arange(n, dtype=np.int64)), flat(k)]
    b = ops.Batch.upload(ctx, vecs, n)
    out, counts = ops.radix_partition(ctx, b, [1], bits)
    check_partition(out, counts, logical(vecs, n), [(k, None)], bits, 0)
    if skew == "one_partition":
        assert counts[-1] == n
    else:
        assert counts[1] == 0 and (np.delete(counts, 1) > 0).all()


@pytest.mark.parametrize("shape", ["staged_i32", "staged_i64", "reg1", "reg2", "reg3", "reg4"])
@pytest.mark.parametrize("bulk", ["0", "1"])
def test_partition_scatter_peer(ctx, monkeypatch, shape, bulk):
    """the PEER = true kernels through b200_partition_scatter with local destination buffers: partition p's rows land
    in buffer p from its offset, nothing before the offset or past the rows changes"""
    import torch
    monkeypatch.setenv("B200_PART_BULK", bulk)
    rng = np.random.default_rng(["staged_i32", "staged_i64", "reg1", "reg2", "reg3", "reg4"].index(shape) * 2 + int(bulk))
    n, bits = 150_001, 2
    if shape.startswith("staged"):
        kd = np.int32 if shape == "staged_i32" else np.int64
        vals = [random_values(rng, kd, n), np.arange(n, dtype=np.int64), random_values(rng, np.int16, n)]
        key_col, rid_col = 0, 1
    else:
        nc = int(shape[3])
        vals = [random_values(rng, np.int64, n), np.arange(n, dtype=np.int64), random_values(rng, np.float64, n),
                random_values(rng, np.uint64, n)][:nc]
        key_col, rid_col = 0, (1 if nc > 1 else None)
    ncols = len(vals)
    b = ops.Batch.upload(ctx, [flat(v) for v in vals], n)
    ids = P.radix_partition_ids(P.hash_columns([(vals[key_col], None)]), bits)
    want = np.bincount(ids, minlength=4)
    starts = [3, 0, 1, 2]
    guard = 64
    sentinel = 0x5A
    bufs = [[torch.full(((starts[p] + int(want[p]) + guard) * v.itemsize,), sentinel, dtype=torch.uint8,
                        device="cuda:0") for v in vals] for p in range(4)]
    dst = [bufs[p][c].data_ptr() for p in range(4) for c in range(ncols)]
    traced_args = (ctx, b, [key_col], bits, dst, starts)
    _, names = traced_window(lambda: (ops.partition_scatter(*traced_args), torch.cuda.synchronize()), [])
    if shape == "staged_i32":
        assert_ran(names, "part_move_staged_kernel<true, false>")
    elif shape == "staged_i64":
        assert_ran(names, "part_move_staged_kernel<true, true>")
        assert_not_ran(names, "part_move_reg_kernel")
    else:
        assert_ran(names, f"part_move_reg_kernel<true, {ncols}, {'true' if bulk == '1' else 'false'}>")
    for p in range(4):
        s, c = starts[p], int(want[p])
        got = [bufs[p][j].cpu().numpy().view(vals[j].dtype) for j in range(ncols)]
        for j in range(ncols):
            raw = bufs[p][j].cpu().numpy()
            w = vals[j].itemsize
            assert (raw[:s * w] == sentinel).all() and (raw[(s + c) * w:] == sentinel).all(), (p, j)
        if rid_col is None:
            np.testing.assert_array_equal(np.sort(got[0][s:s + c]), np.sort(vals[0][ids == p]))
        else:
            rid = got[rid_col][s:s + c]
            np.testing.assert_array_equal(np.sort(rid), np.nonzero(ids == p)[0])
            for j in range(ncols):
                np.testing.assert_array_equal(got[j][s:s + c], vals[j][rid])


def test_partition_int128_rejected(ctx):
    """the partition moves values of at most 8 bytes: an INT128 column is rejected by the radix partition (fast and
    generic shape) and by the shuffle's count and scatter calls"""
    import torch
    rng = np.random.default_rng(129)
    n = 1000
    key = torch.from_numpy(np.arange(n, dtype=np.int64)).to("cuda:0")
    big = int128_column(n, rng)
    b = ops.Batch.wrap(ctx, [(key.data_ptr(), capi.INT64), (big.data_ptr(), capi.INT128)], n, keepalive=[key, big])
    dst_bufs = [torch.zeros(16 * n, dtype=torch.uint8, device="cuda:0") for _ in range(8)]
    dst = [t.data_ptr() for t in dst_bufs]
    offsets = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    dropped = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    counts = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    calls = [lambda: ops.radix_partition(ctx, b, [0], 2), lambda: ops.radix_partition(ctx, b, [0], 8),
             lambda: ops.partition_count(ctx, b, [0], 2), lambda: ops.partition_scatter(ctx, b, [0], 2, dst, [0] * 4),
             lambda: ops.partition_count_dev(ctx, b, [0], 2, counts.data_ptr()),
             lambda: ops.partition_scatter_dev(ctx, b, [0], 2, dst, offsets.data_ptr(), n, dropped.data_ptr())]
    for i, call in enumerate(calls):
        with pytest.raises(capi.B200Error) as e:
            call()
        assert e.value.code == capi.ERR_INVALID, i
    torch.cuda.synchronize()
