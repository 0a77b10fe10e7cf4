"""The in-order MARK probe (b200_join_probe_mark, join_mark.cu) against exact references, and against the kernel trace.

Every case compares, for every probe row in order, the mark byte and its validity bit with a numpy reference and (up
to a few thousand rows) with oracle.port's MARK join: TRUE on a match; NULL for a NULL probe key, or for a key without
a match when the build side holds a NULL key; FALSE otherwise, and for every row when the build side is empty.  The
output buffers are caller-owned, filled with a sentinel and longer than the result, so a write past row n - 1 (or past
the last 32-bit validity word the rows need) shows up as a changed sentinel."""
import zlib

import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran
from oracle import port as P
from test_gpu_agg_kernel_paths import traced_window
from test_gpu_join_kernels import composite_data, dictionary_of

pytestmark = pytest.mark.gpu

# kernel (the __global__ names of join_mark.cu) -> the tests here that assert it ran
KERNEL_CASES = {
    "join_mark_tile_kernel": ["test_single_key", "test_build_sides", "test_large_batches"],
    "join_mark_kernel": ["test_build_sides", "test_composite_keys", "test_unaligned_keys"],
}
KERNEL_EXCLUDED = {}

MARGIN = 64
SENTINEL8 = 0xA5
SENTINEL32 = 0xDEADBEEF
INT_DTYPES = [np.int8, np.uint8, np.int16, np.int32, np.uint32, np.int64, np.uint64]


# ------------------------------------------------------------------ references
def canonical(v):
    """equality classes of join keys: -0.0 == +0.0, every NaN equal"""
    v = np.asarray(v)
    if v.dtype.kind != "f":
        return v
    v = np.where(v == 0, np.zeros(1, v.dtype), v)
    bits = v.view(np.uint64 if v.itemsize == 8 else np.uint32).copy()
    bits[np.isnan(v)] = 0x7FF8000000000000 if v.itemsize == 8 else 0x7FC00000
    return bits


def numpy_mark(bvals, bvalid, pvals, pvalid):
    """single key column: (mark, valid) per probe row"""
    hit = np.isin(canonical(pvals), canonical(bvals)[bvalid]) & pvalid
    if len(bvals) == 0:
        return hit, np.ones(len(pvals), dtype=bool)
    return hit, hit | (pvalid & bool(bvalid.all()))


# ------------------------------------------------------------------ running a probe
class MarkRun:
    """create, sink, finalize, probe_mark into sentinel-filled caller-owned buffers"""

    def __init__(self, key_types, builds, probe, n):
        self.key_types, self.builds, self.probe, self.n = key_types, builds, probe, n

    def __call__(self, ctx):
        import torch
        nk = len(self.key_types)
        j = ops.HashJoin(ctx, capi.JOIN_MARK, self.key_types, [])
        for b in self.builds:
            j.sink(b, list(range(nk)), [])
        j.finalize()
        mark = torch.full((self.n + MARGIN,), SENTINEL8, dtype=torch.uint8, device="cuda:0")
        words32 = (self.n + 31) // 32
        valid = torch.full((words32 + MARGIN,), SENTINEL32 - (1 << 32), dtype=torch.int32, device="cuda:0")
        assert j.probe_mark(self.probe, list(range(nk)), mark.data_ptr(), valid.data_ptr()) is None
        torch.cuda.synchronize()
        j.close()
        return mark.cpu().numpy(), valid.cpu().numpy().view(np.uint32)


def seed(*parts):
    return zlib.crc32(repr(parts).encode())


def check_mark(ctx, key_types, builds, probe, n, exp_mark, exp_valid, kernel):
    """-> kernel names of a traced run in which `kernel` (the variant the case means to reach) was recorded, after
    comparing every row and the sentinels"""
    (mark, words), names = traced_window(lambda: MarkRun(key_types, builds, probe, n)(ctx), [kernel])
    words32 = (n + 31) // 32
    assert (mark[n:] == SENTINEL8).all(), "mark written past the last row"
    assert (words[words32:] == SENTINEL32).all(), "validity written past the last word"
    got_valid = np.unpackbits(words[:words32].view(np.uint8), bitorder="little")[:n].astype(bool)
    bad = np.flatnonzero(got_valid != exp_valid)
    assert bad.size == 0, ("validity differs at rows", bad[:10], got_valid[bad[:10]], exp_valid[bad[:10]])
    bad = np.flatnonzero(mark[:n] != exp_mark.astype(np.uint8))
    assert bad.size == 0, ("mark differs at rows", bad[:10], mark[bad[:10]], exp_mark[bad[:10]])
    return names


def upload(ctx, vectors, n):
    return ops.Batch.upload(ctx, vectors, n)


def key_data(rng, dtype, nb, n, dups=False):
    """build keys (unique unless dups) and probe keys of which about half hit; floats get -0.0 / +0.0 and NaN on both
    sides"""
    dtype = np.dtype(dtype)
    if dtype.kind == "f":
        pool = np.concatenate([np.arange(-3000, 3000, dtype=dtype) / 4, np.array([np.nan, -np.inf, np.inf], dtype)])
        pool = pool[pool != 0]
        b = rng.choice(pool, size=nb, replace=dups)
        b[:2] = [-0.0, np.nan]
        p = np.where(rng.random(n) < 0.5, rng.choice(b, size=n), rng.integers(-9000, 9000, size=n) + 0.125).astype(dtype)
        special = rng.random(n)
        p[special < 0.05] = 0.0                                    # matches the build side's -0.0
        p[(special >= 0.05) & (special < 0.1)] = np.nan
        return b, p
    info = np.iinfo(dtype)
    span = min(int(info.max) - int(info.min) + 1, 4 * max(nb, 1))
    lo = int(info.min) if dtype.itemsize == 1 else max(int(info.min), -span // 2 if info.min < 0 else 0)
    universe = np.arange(lo, lo + span, dtype=np.int64)
    b = rng.choice(universe, size=nb, replace=dups or nb > len(universe)).astype(dtype)
    p = rng.choice(universe, size=n).astype(dtype)
    return b, p


def dense_expected(dtype, bvals, bvalid, no_dense):
    """b200_join_finalize's choice of the direct-addressed table for these build keys"""
    k = bvals[bvalid]
    if no_dense or np.dtype(dtype).kind == "f" or len(k) == 0 or len(np.unique(k)) != len(k):
        return False
    rng = int(k.max()) - int(k.min()) + 1
    return rng <= max(8 * len(bvals), 1 << 20) and rng <= 1 << 28


# ------------------------------------------------------------------ single key, flat aligned: the tile kernel
@pytest.mark.parametrize("n", [1, 2047, 2049, 100003])
@pytest.mark.parametrize("table", ["dense", "hash"])
@pytest.mark.parametrize("dtype", INT_DTYPES + [np.float32, np.float64])
def test_single_key(ctx, monkeypatch, dtype, table, n):
    """1-, 2-, 4- and 8-byte integer keys and FLOAT / DOUBLE keys (-0.0, NaN), with NULL probe keys, against numpy and
    the oracle; the tile kernel runs with the template for the key width and the table"""
    if table == "hash":
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(seed(np.dtype(dtype).str, table, n))
    nb = 100 if np.dtype(dtype).itemsize == 1 else 3000
    bvals, pvals = key_data(rng, dtype, nb, n)
    bvalid = np.ones(nb, dtype=bool)
    pvalid = rng.random(n) > 0.1
    build = upload(ctx, [ops.Vector.flat(bvals)], nb)
    probe = upload(ctx, [ops.Vector.flat(pvals, pvalid)], n)
    exp_mark, exp_valid = numpy_mark(bvals, bvalid, pvals, pvalid)
    if n <= 2049:
        om, ov = P.hash_join([(bvals, bvalid)], [(pvals, pvalid)], nb, n, "mark")
        assert np.array_equal(om, exp_mark) and np.array_equal(ov, exp_valid)
    names = check_mark(ctx, [capi.TYPE_OF_DTYPE[np.dtype(dtype)]], [build], probe, n, exp_mark, exp_valid,
                       "join_mark_tile_kernel")
    fast8 = np.dtype(dtype) in (np.dtype(np.int64), np.dtype(np.uint64))
    dense = dense_expected(dtype, bvals, bvalid, table == "hash")
    assert dense == (table == "dense" and np.dtype(dtype).kind != "f")
    assert_ran(names, f"join_mark_tile_kernel<{str(fast8).lower()}, {str(dense).lower()}>")
    assert_not_ran(names, "join_mark_kernel", "join_probe_kernel", "join_probe_tile_kernel")


# ------------------------------------------------------------------ build sides and probe vector shapes
BUILDS = ["dups", "null_key", "only_null", "empty", "split"]


@pytest.mark.parametrize("shape", ["flat", "const", "null_const", "dict"])
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("dtype", [np.int32, np.int64, np.float64])
def test_build_sides(ctx, dtype, build, shape):
    """duplicate build keys, a build side with a NULL key, one of only NULL keys, an empty one, one sunk in two batches;
    flat (tile kernel), constant and dictionary (generic kernel) probe vectors"""
    rng = np.random.default_rng(seed(np.dtype(dtype).str, build, shape))
    n, nb = 2049, 1500
    bvals, pvals = key_data(rng, dtype, nb, n, dups=build == "dups")
    if build == "dups":
        bvals[nb // 2:] = bvals[:nb - nb // 2]
    bvalid = np.ones(nb, dtype=bool)
    if build == "null_key":
        bvalid[7] = False
    if build == "only_null":
        bvalid[:] = False
    if build == "empty":
        bvals, bvalid, nb = bvals[:0], bvalid[:0], 0
    pvalid = rng.random(n) > 0.1
    if shape == "flat":
        pv = ops.Vector.flat(pvals, pvalid)
    elif shape in ("const", "null_const"):
        pv = ops.Vector.constant(bvals[3] if nb else pvals[0], dtype, is_null=shape == "null_const")
    else:
        pv = dictionary_of(pvals, pvalid, rng)
    pvals_l, pvalid_l = pv.logical(n)
    if build == "split":
        builds = [upload(ctx, [ops.Vector.flat(bvals[:600], bvalid[:600])], 600),
                  upload(ctx, [ops.Vector.flat(bvals[600:], bvalid[600:])], nb - 600)]
    else:
        builds = [upload(ctx, [ops.Vector.flat(bvals, bvalid)], nb)] if nb else []
    exp_mark, exp_valid = numpy_mark(bvals, bvalid, pvals_l, pvalid_l)
    om, ov = P.hash_join([(bvals, bvalid)], [(pvals_l, pvalid_l)], nb, n, "mark")
    assert np.array_equal(om, exp_mark) and np.array_equal(ov, exp_valid)
    if build == "empty":
        assert not exp_mark.any() and exp_valid.all()          # FALSE for every row, NULL keys too
    if build == "only_null":
        assert not exp_valid.any()                             # NULL for every row
    if shape == "const":
        assert exp_mark.all() or build in ("only_null", "empty")
    kernel = "join_mark_tile_kernel" if shape == "flat" else "join_mark_kernel"
    names = check_mark(ctx, [capi.TYPE_OF_DTYPE[np.dtype(dtype)]], builds, upload(ctx, [pv], n), n, exp_mark, exp_valid,
                       kernel)
    if shape == "flat":
        assert_ran(names, "join_mark_tile_kernel")
        assert_not_ran(names, "join_mark_kernel")
    else:
        assert_ran(names, "join_mark_kernel")
        assert_not_ran(names, "join_mark_tile_kernel")
    assert_not_ran(names, "join_probe_kernel", "join_probe_tile_kernel")


@pytest.mark.parametrize("case", ["int64-dense", "int64-hash", "int32-nulls", "float64"])
def test_large_batches(ctx, monkeypatch, case):
    """a few million probe rows (a grid-strided tile loop with several tiles per CTA) against the Q14-like shape"""
    if case == "int64-hash":
        monkeypatch.setenv("B200_JOIN_NO_DENSE", "1")
    rng = np.random.default_rng(seed(case))
    dtype = {"int32-nulls": np.int32, "float64": np.float64}.get(case, np.int64)
    n, nb = 3_000_017, 200_000
    if np.dtype(dtype).kind == "f":
        bvals, pvals = key_data(rng, dtype, 3000, n)
        nb = 3000
    else:
        bvals = (rng.permutation(400_000)[:nb] + 1).astype(dtype)
        pvals = rng.integers(0, 400_002, size=n).astype(dtype)
    bvalid = np.ones(nb, dtype=bool)
    if case == "int32-nulls":
        bvalid[123] = False
    pvalid = rng.random(n) > 0.02 if case == "int32-nulls" else np.ones(n, dtype=bool)
    build = upload(ctx, [ops.Vector.flat(bvals, bvalid if not bvalid.all() else None)], nb)
    probe = upload(ctx, [ops.Vector.flat(pvals, pvalid if not pvalid.all() else None)], n)
    exp_mark, exp_valid = numpy_mark(bvals, bvalid, pvals, pvalid)
    names = check_mark(ctx, [capi.TYPE_OF_DTYPE[np.dtype(dtype)]], [build], probe, n, exp_mark, exp_valid,
                       "join_mark_tile_kernel")
    # INTEGER keys 1 .. 400 000 with a NULL among them still make a direct-addressed table
    assert_ran(names, {"int64-dense": "join_mark_tile_kernel<true, true>", "int64-hash": "join_mark_tile_kernel<true, false>",
                       "int32-nulls": "join_mark_tile_kernel<false, true>",
                       "float64": "join_mark_tile_kernel<false, false>"}[case])


# ------------------------------------------------------------------ the generic kernel
@pytest.mark.parametrize("shape", ["flat", "dict"])
@pytest.mark.parametrize("nkeys", [2, 4])
def test_composite_keys(ctx, nkeys, shape):
    """composite keys, with forced 64-bit hash collisions, keys hashing to the empty-slot key, duplicates and NULLs in
    every position (test_gpu_join_kernels.composite_data), against the oracle"""
    rng = np.random.default_rng(700 + nkeys + (shape == "dict"))
    nb, n = 300, 2049
    bk, pk = composite_data(rng, nkeys, nb, n)
    bt = [capi.TYPE_OF_DTYPE[np.asarray(v).dtype] for v, _ in bk]
    build = upload(ctx, [ops.Vector.flat(v, ok) for v, ok in bk], nb)
    pvs = [ops.Vector.flat(v, ok) if shape == "flat" else dictionary_of(v, ok, rng) for v, ok in pk]
    exp_mark, exp_valid = P.hash_join(bk, pk, nb, n, "mark")
    assert exp_mark.any() and (~exp_valid).any()   # the build side holds NULL keys: no row is FALSE
    names = check_mark(ctx, bt, [build], upload(ctx, pvs, n), n, exp_mark, exp_valid, "join_mark_kernel")
    assert_ran(names, "join_mark_kernel")
    assert_not_ran(names, "join_mark_tile_kernel", "join_probe_kernel")


@pytest.mark.parametrize("n", [1, 2047, 2049])
def test_unaligned_keys(ctx, n):
    """a flat key column that does not start on 16 bytes cannot be bulk-copied: the generic kernel takes it"""
    import torch
    rng = np.random.default_rng(n)
    nb = 500
    bvals, pvals = key_data(rng, np.int64, nb, n)
    build = upload(ctx, [ops.Vector.flat(bvals)], nb)
    dev = torch.from_numpy(np.concatenate([pvals[:1], pvals])).to("cuda:0")
    probe = ops.Batch.wrap(ctx, [(dev.data_ptr() + 8, capi.INT64)], n, keepalive=dev)
    exp_mark, exp_valid = numpy_mark(bvals, np.ones(nb, bool), pvals, np.ones(n, bool))
    names = check_mark(ctx, [capi.INT64], [build], probe, n, exp_mark, exp_valid, "join_mark_kernel")
    assert_ran(names, "join_mark_kernel")
    assert_not_ran(names, "join_mark_tile_kernel")


# ------------------------------------------------------------------ the entry point's contract
def test_same_marks_as_the_generic_mark_probe(ctx):
    """b200_join_probe(MARK) returns the same marks in an unspecified order: put them back by lhs_sel and compare"""
    import torch
    rng = np.random.default_rng(5)
    n, nb = 50_000, 4000
    bvals, pvals = key_data(rng, np.int64, nb, n)
    bvalid = np.ones(nb, dtype=bool)
    bvalid[1] = False
    pvalid = rng.random(n) > 0.1
    j = ops.HashJoin(ctx, capi.JOIN_MARK, [capi.INT64], [])
    j.sink(upload(ctx, [ops.Vector.flat(bvals, bvalid)], nb), [0], [])
    j.finalize()
    probe = upload(ctx, [ops.Vector.flat(pvals, pvalid)], n)
    mark, valid = j.probe_mark(probe, [0])
    sel = torch.empty(n, dtype=torch.int32, device="cuda:0")
    out, count = j.execute(probe, [0], [], 0, sel.data_ptr())
    old_mark, old_valid = out.download(0)
    order = sel.cpu().numpy()
    assert count == n and sorted(order.tolist()) == list(range(n))
    assert np.array_equal(mark[order], old_mark.astype(np.uint8)) and np.array_equal(valid[order], old_valid)
    j.close()


def test_rejects_other_joins(ctx):
    """a join of another type, a join not yet finalized, key columns of the wrong type: B200_ERR_INVALID"""
    import torch
    n = 10
    probe = upload(ctx, [ops.Vector.flat(np.arange(n, dtype=np.int64)), ops.Vector.flat(np.arange(n, dtype=np.int32))], n)
    buf = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    for jt in (capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI):
        j = ops.HashJoin(ctx, jt, [capi.INT64], [])
        j.finalize()
        with pytest.raises(capi.B200Error) as e:
            j.probe_mark(probe, [0], buf.data_ptr(), buf.data_ptr() + 256)
        assert e.value.code == capi.ERR_INVALID and "B200_JOIN_MARK" in str(e.value)
        j.close()
    j = ops.HashJoin(ctx, capi.JOIN_MARK, [capi.INT64], [])
    with pytest.raises(capi.B200Error) as e:
        j.probe_mark(probe, [0], buf.data_ptr(), buf.data_ptr() + 256)
    assert e.value.code == capi.ERR_INVALID and "finalize" in str(e.value)
    j.finalize()
    with pytest.raises(capi.B200Error) as e:
        j.probe_mark(probe, [1], buf.data_ptr(), buf.data_ptr() + 256)
    assert e.value.code == capi.ERR_INVALID and "type" in str(e.value)
    # an empty probe batch is a no-op
    empty = upload(ctx, [ops.Vector.flat(np.zeros(0, dtype=np.int64))], 0)
    assert j.probe_mark(empty, [0], buf.data_ptr(), buf.data_ptr() + 256) is None
    j.close()
