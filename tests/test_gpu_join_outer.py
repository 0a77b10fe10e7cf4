"""RIGHT and FULL OUTER hash joins (B200_JOIN_RIGHT / B200_JOIN_OUTER): the probe kernels' build-row match flags and
b200_join_scan_unmatched, against exact references and against the kernel trace.

The reference is the oracle's equality join: a RIGHT join's probe returns the INNER pairs and a FULL join's the LEFT
pairs (oracle.port.hash_join), and the scan returns, in build-row order, every build row that no probe pair names -
NULL-key build rows included.  Every case gives the build side a row-id payload column where it can, so the whole
result compares as rows of (probe row, lhs cells, payload cells).  Row-id and lhs_sel buffers are caller-owned, filled
with a sentinel and longer than the result, so a write past the count shows up.  A subset is also checked against the
reference DuckDB's own RIGHT / FULL join."""
import ctypes as C
import zlib

import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran
from oracle import port as P
from test_gpu_agg_kernel_paths import traced_window
from test_gpu_join_kernels import cells, composite_data, flat, random_values
from test_gpu_join_mark import key_data

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of join_outer.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "join_rows_offset_kernel": ["test_scan_ranges", "test_build_sides"],
}
KERNEL_EXCLUDED = {}

JT = {"right": capi.JOIN_RIGHT, "full": capi.JOIN_OUTER}
SENTINEL = 0xDEADBEEF
MARGIN = 256


def seed(*parts):
    return zlib.crc32(repr(parts).encode())


def sentinel_buffer(length):
    import torch
    return torch.full((max(1, length) + MARGIN,), SENTINEL - (1 << 32), dtype=torch.int32, device="cuda:0")


def download(batch):
    from test_gpu_kernel_paths import _download_raw
    return _download_raw(batch)


# ------------------------------------------------------------------ reference
def expected(jt, bkeys, pkey_batches, nb):
    """-> (probe pairs per probe batch, the set of matched build rows).  Pairs: (probe row, build row or -1)."""
    per_batch, matched = [], set()
    for pkeys, npb in pkey_batches:
        pairs = P.hash_join(bkeys, pkeys, nb, npb, "inner" if jt == "right" else "left")
        matched.update(b for _, b in pairs if b >= 0)
        per_batch.append(pairs)
    return per_batch, matched


# ------------------------------------------------------------------ running a join
class OuterRun:
    """create, sink every build batch, finalize, probe every probe batch (lhs_sel into sentinel buffers), then scan
    every range (build row ids into sentinel buffers)"""

    def __init__(self, jt, key_types, pay_types, builds, nkeys, probes, nlhs, ranges, capacity=0):
        self.jt, self.key_types, self.pay_types, self.builds = jt, key_types, pay_types, builds
        self.nkeys, self.probes, self.nlhs, self.ranges, self.capacity = nkeys, probes, nlhs, ranges, capacity

    def __call__(self, ctx):
        import torch
        j = ops.HashJoin(ctx, JT[self.jt], self.key_types, self.pay_types)
        npay = len(self.pay_types)
        for b in self.builds:
            j.sink(b, list(range(self.nkeys)), list(range(self.nkeys, self.nkeys + npay)))
        j.finalize()
        probed, codes = [], []
        for batch, sel_len in self.probes:
            sel = sentinel_buffer(sel_len)
            keys, lhs = list(range(self.nkeys)), list(range(self.nkeys, self.nkeys + self.nlhs))
            try:
                out, count = j.execute(batch, keys, lhs, self.capacity, sel.data_ptr())
            except capi.B200Error as e:
                codes.append(e.code)            # LEFT-style capacity overflow: retry sized by the counting pass
                out, count = j.execute(batch, keys, lhs, 0, sel.data_ptr())
            probed.append((count, download(out), sel.cpu().numpy().view(np.uint32).copy()))
            out.free()
        scanned = []
        for b, e in self.ranges:
            rows = sentinel_buffer(e - b)
            out, count = C.c_void_p(), C.c_uint64()
            capi.check(capi.lib().b200_join_scan_unmatched(j.handle, b, e, C.byref(out), C.c_void_p(rows.data_ptr()),
                                                           C.byref(count)))
            batch = ops.Batch(ctx, out)
            assert batch.nrows == count.value and batch.ncols == npay
            scanned.append((count.value, download(batch), rows.cpu().numpy().view(np.uint32).copy()))
            batch.free()
        torch.cuda.synchronize()
        j.close()
        return probed, scanned, codes


def check_outer(ctx, jt, key_types, pay_types, builds, probes, nkeys, nlhs, ranges, kernel, capacity=0):
    """run the join in a traced window and compare with the reference -> (kernel names, retry codes).
    builds: [(Batch, logical columns: keys, then payload)]; probes: [(Batch, logical columns: keys, then lhs, n)]."""
    bcols = [(np.concatenate([c[i][0] for _, c in builds]), np.concatenate([c[i][1] for _, c in builds]))
             for i in range(nkeys + len(pay_types))] if builds else \
        [(np.zeros(0, capi.DTYPE_OF_TYPE[t]), np.zeros(0, bool)) for t in key_types + pay_types]
    nb = len(bcols[0][0])
    pairs, matched = expected(jt, bcols[:nkeys], [(pc[:nkeys], n) for _, pc, n in probes], nb)
    pay = [cells(v, ok) for v, ok in bcols[nkeys:]]
    run = OuterRun(jt, key_types, pay_types, [b for b, _ in builds], nkeys,
                   [(b, len(p) + 1) for (b, _, _), p in zip(probes, pairs)], nlhs, ranges, capacity)
    (probed, scanned, codes), names = traced_window(lambda: run(ctx), [kernel])
    for (count, res, sel), p, (_, pcols, n) in zip(probed, pairs, probes):
        lhs = [cells(v, ok) for v, ok in pcols[nkeys:nkeys + nlhs]]
        exp = sorted(((r, tuple(c[r] for c in lhs), tuple(c[b] if b >= 0 else None for c in pay)) for r, b in p),
                     key=repr)
        assert count == len(exp), (count, len(exp))
        assert (sel[count:] == SENTINEL).all(), "lhs_sel was written past the result"
        got_cols = [cells(v, ok) for v, ok in res]
        assert len(got_cols) == nlhs + len(pay_types)
        got = sorted(((int(sel[i]), tuple(c[i] for c in got_cols[:nlhs]), tuple(c[i] for c in got_cols[nlhs:]))
                      for i in range(count)), key=repr)
        assert got == exp, next(((g, e) for g, e in zip(got, exp) if g != e), None)
    for (count, res, rows), (b, e) in zip(scanned, ranges):
        exp_rows = [r for r in range(b, e) if r not in matched]
        assert count == len(exp_rows), ((b, e), count, len(exp_rows))
        assert rows[:count].tolist() == exp_rows, (b, e)      # build-row order
        assert (rows[count:] == SENTINEL).all(), "build row ids written past the result"
        got_cols = [cells(v, ok) for v, ok in res]
        for c, pc in zip(got_cols, pay):
            assert c == [pc[r] for r in exp_rows], (b, e)
    return names, codes


def upload(ctx, vectors, n):
    return ops.Batch.upload(ctx, vectors, n), [v.logical(n) for v in vectors]


def full_range(nb):
    return [(0, nb)]


# ------------------------------------------------------------------ single key: the tile probe
@pytest.mark.parametrize("table", ["dense", "hash"])
@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.uint16, np.int32, np.int64, np.uint64, np.float32, np.float64])
@pytest.mark.parametrize("jt", list(JT))
def test_single_key(ctx, monkeypatch, jt, dtype, table):
    """1-, 2-, 4- and 8-byte integer keys and FLOAT / DOUBLE keys (-0.0, NaN), a NULL build key and NULL probe keys,
    nullable payloads; the tile probe runs (never a lean kernel, which flags no build row), the scan compacts through
    the filter's tile mask kernel and its generic compaction (the payload is nullable)"""
    if table == "hash":
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(seed(jt, np.dtype(dtype).str, table))
    nb = 100 if np.dtype(dtype).itemsize == 1 else 3000
    n = 4099
    bvals, pvals = key_data(rng, dtype, nb, n)
    bvalid = np.ones(nb, dtype=bool)
    bvalid[5] = False
    pvalid = rng.random(n) > 0.1
    rid = np.arange(nb, dtype=np.int64)
    p4 = random_values(rng, np.int32, nb)
    p4ok = rng.random(nb) > 0.2
    lhs = random_values(rng, np.int64, n)
    builds = [upload(ctx, [flat(bvals, bvalid), flat(rid), flat(p4, p4ok)], nb)]
    pb, pcols = upload(ctx, [flat(pvals, pvalid), flat(lhs)], n)
    kt = capi.TYPE_OF_DTYPE[np.dtype(dtype)]
    names, _ = check_outer(ctx, jt, [kt], [capi.INT64, capi.INT32], builds, [(pb, pcols, n)], 1, 1, full_range(nb),
                           "join_probe_tile_kernel")
    # probe keys with NULLs: never the 8-byte specialisation
    assert_ran(names, "join_probe_tile_kernel<false, false>", "filter_mask_tile_kernel", "compact_kernel")
    assert_not_ran(names, "join_probe_lean2_kernel", "join_probe_tile_kernel<true, true>", "join_probe_kernel<1>",
                   "join_rows_offset_kernel")
    if table == "dense" and np.dtype(dtype).kind != "f":
        assert_ran(names, "join_dense_build_kernel")


@pytest.mark.parametrize("table", ["dense", "hash"])
@pytest.mark.parametrize("jt", list(JT))
def test_inline_payload_shape(ctx, monkeypatch, jt, table):
    """Q14's shape: unique BIGINT keys and a 1-byte payload without NULLs, which an INNER join keeps inline in the
    table.  A RIGHT / FULL join must still find the build row: the dense table keeps row ids, the hash table its head
    row.  The scan's payload is NULL-free: the filter's tile compaction runs."""
    if table == "hash":
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(seed("inline", jt, table))
    nb, n = 5000, 20011
    bk = (rng.permutation(10000)[:nb] + 1).astype(np.int64)
    pay = (np.arange(nb) % 251).astype(np.uint8)
    pk = rng.integers(0, 10002, size=n).astype(np.int64)
    lhs = random_values(rng, np.int64, n)
    builds = [upload(ctx, [flat(bk), flat(pay)], nb)]
    pb, pcols = upload(ctx, [flat(pk), flat(lhs)], n)
    names, _ = check_outer(ctx, jt, [capi.INT64], [capi.UINT8], builds, [(pb, pcols, n)], 1, 1, full_range(nb),
                           "join_probe_tile_kernel")
    assert_ran(names, "join_probe_tile_kernel<true, false>", "compact_tile_kernel")
    assert_not_ran(names, "join_probe_lean2_kernel", "join_probe_tile_kernel<true, true>", "join_inline_kernel"
                   if table == "dense" else "join_probe_kernel<1>")


# ------------------------------------------------------------------ build sides, several sinks and probes, ranges
BUILDS = ["dups", "null_keys", "empty_build", "empty_probe", "all_matched"]


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("jt", list(JT))
def test_build_sides(ctx, jt, build):
    """duplicate build keys, NULL build keys, an empty build side, an empty probe side, a build side every row of
    which is matched; the build sunk in three batches and probed in three, the flags accumulating across probes;
    the scan over every row and over a range that starts past row 0"""
    rng = np.random.default_rng(seed("sides", jt, build))
    nb = 0 if build == "empty_build" else 1000
    bvals = rng.integers(0, 800, size=nb).astype(np.int32)
    if build == "dups":
        bvals[nb // 2:] = bvals[:nb - nb // 2]
    if build == "all_matched":
        bvals = np.arange(nb, dtype=np.int32)
    bvalid = np.ones(nb, dtype=bool)
    if build in ("null_keys", "dups"):
        bvalid[rng.random(nb) < 0.05] = False
    rid = np.arange(nb, dtype=np.int64)
    cuts = [0, nb // 3, 2 * nb // 3, nb]
    builds = [upload(ctx, [flat(bvals[a:b], bvalid[a:b]), flat(rid[a:b])], b - a) for a, b in zip(cuts, cuts[1:])
              if b > a]
    probes = []
    for n in ([0] if build == "empty_probe" else [700, 2049, 333]):
        pv = rng.integers(0, 1000, size=n).astype(np.int32)
        pok = rng.random(n) > 0.1
        if build == "all_matched" and n == 2049:
            pv[:nb], pok[:nb] = np.arange(nb, dtype=np.int32), True
        lhs = random_values(rng, np.float64, n)
        b, c = upload(ctx, [flat(pv, pok), flat(lhs, rng.random(n) > 0.3)], n)
        probes.append((b, c, n))
    ranges = [(0, nb)] + ([(64, nb)] if nb > 64 else [])
    names, _ = check_outer(ctx, jt, [capi.INT32], [capi.INT64], builds, probes, 1, 1, ranges,
                           "filter_mask_tile_kernel" if nb else "join_probe_tile_kernel")
    if build == "all_matched":
        assert_not_ran(names, "compact_tile_kernel", "compact_kernel")   # nothing to compact
    elif nb > 64:
        assert_ran(names, "join_rows_offset_kernel")


def test_scan_ranges(ctx):
    """ranges whose ends fall at 0, 63, 64, 65 and the last row, scanned in any order and more than once (the scan
    reads the flags, it does not clear them)"""
    rng = np.random.default_rng(11)
    nb, n = 1000, 3000
    bvals = rng.integers(0, 1500, size=nb).astype(np.int64)
    rid = np.arange(nb, dtype=np.int64)
    builds = [upload(ctx, [flat(bvals), flat(rid)], nb)]
    pv = rng.integers(0, 1500, size=n).astype(np.int64)
    pb, pc = upload(ctx, [flat(pv)], n)
    ranges = [(0, 0), (0, 63), (0, 64), (0, 65), (64, 64), (64, 65), (64, 128), (960, 999), (960, nb), (0, nb),
              (nb // 64 * 64, nb), (0, 63)]
    names, _ = check_outer(ctx, "right", [capi.INT64], [capi.INT64], builds, [(pb, pc, n)], 1, 0, ranges,
                           "join_rows_offset_kernel")
    assert_ran(names, "join_rows_offset_kernel", "compact_tile_kernel")


# ------------------------------------------------------------------ composite keys: the generic probe
@pytest.mark.parametrize("nkeys", [2, 4])
@pytest.mark.parametrize("jt", list(JT))
def test_composite_keys(ctx, jt, nkeys):
    """composite keys with forced 64-bit hash collisions, keys hashing to the side slot, duplicates and NULLs in every
    position (test_gpu_join_kernels.composite_data): the generic probe with its counting pass flags the rows"""
    rng = np.random.default_rng(seed("composite", jt, nkeys))
    nb, npb = 300, 400
    bk, pk = composite_data(rng, nkeys, nb, npb)
    rid = np.arange(nb, dtype=np.int64)
    bt = [capi.TYPE_OF_DTYPE[np.asarray(v).dtype] for v, _ in bk]
    builds = [upload(ctx, [flat(v[:120], ok[:120]) for v, ok in bk] + [flat(rid[:120])], 120),
              upload(ctx, [flat(v[120:], ok[120:]) for v, ok in bk] + [flat(rid[120:])], nb - 120)]
    lhs = random_values(rng, np.int32, npb)
    pb, pcols = upload(ctx, [flat(v, ok) for v, ok in pk] + [flat(lhs)], npb)
    names, _ = check_outer(ctx, jt, bt, [capi.INT64], builds, [(pb, pcols, npb)], nkeys, 1, full_range(nb),
                           "join_probe_kernel")
    assert_ran(names, "join_probe_kernel<0>", "join_probe_kernel<1>")
    assert_not_ran(names, "join_probe_tile_kernel")


# ------------------------------------------------------------------ capacity retry, wide payloads
@pytest.mark.parametrize("probe_kind", ["tile", "generic"])
@pytest.mark.parametrize("jt", list(JT))
def test_capacity_retry(ctx, jt, probe_kind):
    """duplicate build keys and an output capacity of one row per probe row: the first call returns
    B200_ERR_CAPACITY after it may have flagged rows, the retry emits the same rows; the scan sees the same flags"""
    rng = np.random.default_rng(seed("capacity", jt, probe_kind))
    nb, n = 2000, 5000
    bvals = np.repeat(np.arange(nb // 8, dtype=np.int64) * 2, 8)     # 0, 2, .., 498, eight rows each
    rid = np.arange(nb, dtype=np.int64)
    builds = [upload(ctx, [flat(bvals), flat(rid)], nb)]
    pv = rng.integers(0, 520, size=n).astype(np.int64)             # about 4 result rows per probe row
    pok = rng.random(n) > 0.05
    if probe_kind == "tile":
        pb, pcols = upload(ctx, [flat(pv, pok)], n)
    else:
        from test_gpu_join_kernels import dictionary_of
        v = dictionary_of(pv, pok, rng)
        pb, pcols = upload(ctx, [v], n)
    names, codes = check_outer(ctx, jt, [capi.INT64], [capi.INT64], builds, [(pb, pcols, n)], 1, 0, full_range(nb),
                               "join_probe_tile_kernel" if probe_kind == "tile" else "join_probe_kernel", capacity=n)
    assert codes == [capi.ERR_CAPACITY]
    assert_ran(names, "join_probe_tile_kernel" if probe_kind == "tile" else "join_probe_kernel<1>")


def test_twelve_payload_columns(ctx):
    """12 payload columns, one more than a filter call projects next to the flags: the scan projects them in two
    slices, which must select the same rows in the same order"""
    rng = np.random.default_rng(12)
    nb, n = 2500, 4000
    bvals = rng.integers(0, 5000, size=nb).astype(np.int32)
    dts = [np.int64, np.int8, np.uint16, np.int32, np.float32, np.float64, np.uint8, np.int16, np.uint32, np.uint64,
           np.int64, np.float64]
    pays = [(random_values(rng, dt, nb), rng.random(nb) > 0.1 if i % 3 == 0 else None) for i, dt in enumerate(dts)]
    pays[0] = (np.arange(nb, dtype=np.int64), None)
    builds = [upload(ctx, [flat(bvals)] + [flat(v, ok) for v, ok in pays], nb)]
    pv = rng.integers(0, 5000, size=n).astype(np.int32)
    pb, pcols = upload(ctx, [flat(pv)], n)
    check_outer(ctx, "full", [capi.INT32], [capi.TYPE_OF_DTYPE[np.dtype(d)] for d in dts], builds, [(pb, pcols, n)],
                1, 0, [(0, nb), (128, 2000)], "filter_mask_tile_kernel")


# ------------------------------------------------------------------ the reference DuckDB's RIGHT / FULL join
@pytest.mark.parametrize("kind", ["RIGHT", "FULL"])
def test_against_duckdb(ctx, kind):
    """the same tables joined by the reference DuckDB: its (probe id, build id) pairs, NULL ids included, equal ours"""
    from oracle import duckdb_ref as R
    if not R.available():
        pytest.skip("needs oracle/_ref/libduckdb_ref.so (built by build())")
    rng = np.random.default_rng(seed("duckdb", kind))
    nb, n = 3000, 20000
    bk = rng.integers(0, 4000, size=nb).astype(np.int64)
    bok = rng.random(nb) > 0.03
    pk = rng.integers(0, 6000, size=n).astype(np.int64)
    pok = rng.random(n) > 0.03
    con = R.Connection(threads=2)
    try:
        con.load_table("b", {"bid": np.arange(nb, dtype=np.int64), "k": (bk, bok)})
        con.load_table("p", {"pid": np.arange(n, dtype=np.int64), "k": (pk, pok)})
        theirs = sorted(con.fetchall(f"SELECT p.pid, b.bid FROM p {kind} JOIN b ON p.k = b.k"),
                        key=lambda r: (r[0] is None, r[0] or 0, r[1] is None, r[1] or 0))
    finally:
        con.close()
    j = ops.HashJoin(ctx, JT["right" if kind == "RIGHT" else "full"], [capi.INT64], [capi.INT64])
    j.sink(ops.Batch.upload(ctx, [flat(bk, bok), flat(np.arange(nb, dtype=np.int64))], nb), [0], [1])
    j.finalize()
    out, count = j.execute(ops.Batch.upload(ctx, [flat(pk, pok), flat(np.arange(n, dtype=np.int64))], n), [0], [1])
    (pid, _), (bid, bvalid) = download(out)
    ours = [(int(p), int(b) if ok else None) for p, b, ok in zip(pid[:count], bid[:count], bvalid[:count])]
    scan, scount, rows = j.scan_unmatched(want_rows=True)
    (sbid, _), = download(scan)
    assert sbid[:scount].tolist() == rows.tolist()
    ours += [(None, int(b)) for b in rows]
    j.close()
    ours.sort(key=lambda r: (r[0] is None, r[0] or 0, r[1] is None, r[1] or 0))
    assert ours == theirs


# ------------------------------------------------------------------ the entry point's contract
def test_rejects(ctx):
    """a join of another type, one not yet finalized, a range that does not start on 64 rows or leaves the build
    side: B200_ERR_INVALID"""
    nb = 200
    b = ops.Batch.upload(ctx, [flat(np.arange(nb, dtype=np.int64))], nb)
    for jt in (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_MARK):
        j = ops.HashJoin(ctx, jt, [capi.INT64], [])
        j.sink(b, [0], [])
        j.finalize()
        with pytest.raises(capi.B200Error) as e:
            j.scan_unmatched()
        assert e.value.code == capi.ERR_INVALID and "B200_JOIN_RIGHT" in str(e.value)
        j.close()
    j = ops.HashJoin(ctx, capi.JOIN_RIGHT, [capi.INT64], [])
    j.sink(b, [0], [])
    with pytest.raises(capi.B200Error) as e:
        j.scan_unmatched(0, nb)
    assert e.value.code == capi.ERR_INVALID and "finalize" in str(e.value)
    j.finalize()
    for lo, hi in [(1, 10), (63, 100), (64, 63), (0, nb + 1), (256, 300)]:
        with pytest.raises(capi.B200Error) as e:
            j.scan_unmatched(lo, hi)
        assert e.value.code == capi.ERR_INVALID and "range" in str(e.value), (lo, hi)
    out, count = j.scan_unmatched()        # no probe ran: every build row, and no payload column
    assert count == nb and out.ncols == 0 and out.nrows == nb
    j.close()
