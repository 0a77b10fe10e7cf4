"""The aggregate's finalize result: one device block, one validity fill, and for results of at most 1 MiB one copy to a
pinned host copy from which every download is served.

Checked here: which kernels and copies a finalize + download_all makes (TPC-H Q1 shape), exact values and validity
bits (integer sums as Python ints, integer AVG as long double(sum) / count, NULL keys, AVG over NULL inputs only), both
sides of the 1 MiB cut, and the edge cases of the host copy: download after the aggregate is destroyed, a result freed
without a download, 0 groups, and the device view of a small result holding the bytes its download returns."""
import contextlib
import ctypes as C
import json
import os
import tempfile
import time

import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import WINDOW_MARGIN_S, _strip
from test_gpu_agg_kernel_paths import assert_same, descs_of, fetch_groups, reference, sink_all

pytestmark = pytest.mark.gpu

HOST_COPY_MAX = 1 << 20   # b200_agg_finalize copies result blocks up to this size to the host


@contextlib.contextmanager
def gpu_trace():
    """with gpu_trace() as ev: ...  -> afterwards ev["kernel"] holds the kernel names, ev["memcpy"] the memcpy kinds
    (e.g. 'Memcpy DtoH (Device -> Pinned)') of the GPU activity inside the block"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    ev = {"kernel": [], "memcpy": []}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(WINDOW_MARGIN_S)
        yield ev
        torch.cuda.synchronize()
        time.sleep(WINDOW_MARGIN_S)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = sorted(json.load(f).get("traceEvents", []), key=lambda e: e.get("ts", 0))
    ev["kernel"].extend(_strip(e["name"]) for e in events if e.get("cat") == "kernel")
    ev["memcpy"].extend(e["name"] for e in events if e.get("cat") == "gpu_memcpy")


def block_bytes(groups, col_bytes, int_avgs):
    """size of the finalize block: columns of col_bytes[c] bytes per group, int_avgs raw [lo, hi, count] triples"""
    span = lambda b: (b + 16 + 15) & ~15
    vwords = ((groups + 63) // 64 + 2) & ~1
    return (sum(span(groups * b) for b in col_bytes) + int_avgs * span(groups * 24) + len(col_bytes) * vwords * 8)


def d2h(ctx):
    return ctx.stats()["d2h_bytes"]


def raw_download(batch, col):
    """(data bytes, validity words) of one column, as b200_batch_download returns them"""
    info = batch.column_info(col)
    n = batch.nrows
    data = np.zeros(n * capi.TYPE_SIZE[info.type], dtype=np.uint8)
    words = np.zeros(max(1, (n + 63) // 64), dtype=np.uint64)
    capi.check(capi.lib().b200_batch_download(batch.ctx.handle, batch.handle, col,
                                              C.c_void_p(data.ctypes.data) if n else None,
                                              C.c_void_p(words.ctypes.data) if n else None))
    return data, words[:(n + 63) // 64]


def device_bytes(ptr, nbytes):
    import torch
    from duckdb_b200.distributed import _DevArray

    if nbytes == 0:
        return np.zeros(0, dtype=np.uint8)
    return torch.as_tensor(_DevArray(ptr, nbytes, "|u1"), device="cuda").cpu().numpy()


# ------------------------------------------------------------------ TPC-H Q1: kernels and copies
Q1_DESC = [(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_SUM, capi.INT64, 1), (capi.AGG_SUM, capi.INT64, 2),
           (capi.AGG_SUM, capi.INT64, 3), (capi.AGG_AVG, capi.INT64, 0), (capi.AGG_AVG, capi.INT64, 1),
           (capi.AGG_AVG, capi.INT64, 4), (capi.AGG_COUNT_STAR, capi.INT64, -1)]
Q1_AGGS = [("sum", 0), ("sum", 1), ("sum", 2), ("sum", 3), ("avg", 0), ("avg", 1), ("avg", 4), ("count_star", -1)]


def test_q1_finalize_one_copy(ctx):
    import torch

    import bench_data as BD

    n = 3_000_000
    q1 = BD.Gen(torch, torch.device("cuda", 0)).q1(n)
    names = ("rf", "ls", "qty", "price", "disc_price", "charge", "disc")
    cols = [q1[k] for k in names]
    types = [capi.UINT8, capi.UINT8] + [capi.INT64] * 5
    batch = ops.Batch.wrap(ctx, [(t.data_ptr(), ty) for t, ty in zip(cols, types)], n, keepalive=cols)
    host = {k: q1[k].cpu().numpy() for k in names}
    rf, ls = host["rf"], host["ls"]
    code = rf.astype(np.int64) * 256 + ls
    uniq, gid = np.unique(code, return_inverse=True)
    inputs = [(host[k], None) for k in ("qty", "price", "disc_price", "charge", "disc")]
    exp = reference([(rf, None), (ls, None)], gid, len(uniq), inputs, Q1_AGGS)

    for attempt in range(3):
        agg = ops.HashAggregate(ctx, [capi.UINT8, capi.UINT8], Q1_DESC)
        agg.sink(batch, [0, 1], [2, 3, 4, 5, 6])
        ctx.sync()
        with gpu_trace() as ev:
            # a kernel of torch's first: the profiler can lose the first activity of a window
            torch.ones(1, device="cuda").add_(1)
            out = agg.finalize()
            out.download_all()
        agg.close()
        ev["kernel"] = [k for k in ev["kernel"] if not k.startswith("at::")]
        # the profiler now and then drops a record from a window: take one in which every kind of activity arrived
        if {"agg_finalize_kernel", "fill_u64_kernel3"} <= set(ev["kernel"]) and any("DtoH" in m for m in ev["memcpy"]):
            break
        out.free()
    assert sorted(ev["kernel"]) == ["agg_finalize_kernel", "fill_u64_kernel3"], ev["kernel"]
    dtoh = [m for m in ev["memcpy"] if "DtoH" in m]
    assert len(dtoh) == 1, ev["memcpy"]
    assert "Pinned" in dtoh[0], dtoh

    # download_all alone: served from the host copy, no copy at all
    s0 = d2h(ctx)
    with gpu_trace() as ev2:
        res = out.download_all()
    assert ev2["memcpy"] == [] and ev2["kernel"] == [], ev2
    assert d2h(ctx) == s0
    assert_same(fetch_groups(out, 2, len(Q1_AGGS)), exp, Q1_AGGS, inputs)
    assert len(res) == 10
    out.free()
    batch.free()


# ------------------------------------------------------------------ exact values and validity
def nullable_case(rng, n=200_000):
    """INT32 keys with NULLs (a NULL-key group), BIGINT and INTEGER inputs with NULLs, one group whose BIGINT input is
    NULL in every row (its SUM and AVG are NULL), a DOUBLE input"""
    ng = 9
    gid = rng.integers(0, ng, size=n)
    kval = (gid * 1000 - 3000).astype(np.int32)
    kvalid = gid != 4
    kval[~kvalid] = rng.integers(-5, 5, size=int((~kvalid).sum())).astype(np.int32)   # NULL key: value is noise
    big = rng.integers(-2 ** 62, 2 ** 62, size=n, dtype=np.int64)
    bvalid = (rng.random(n) > 0.3) & (gid != 7)
    small = rng.integers(-2 ** 31, 2 ** 31, size=n, dtype=np.int64).astype(np.int32)
    svalid = rng.random(n) > 0.5
    dbl = rng.standard_normal(n)
    keys = [(kval, kvalid)]
    inputs = [(big, bvalid), (small, svalid), (dbl, None)]
    aggs = [("sum", 0), ("avg", 0), ("count", 0), ("min", 0), ("max", 0), ("avg", 1), ("sum", 1), ("avg", 2),
            ("count_star", -1)]
    return keys, gid, ng, inputs, aggs


def test_exact_values_and_validity(ctx):
    rng = np.random.default_rng(11)
    keys, gid, ng, inputs, aggs = nullable_case(rng)
    n = len(gid)
    agg = ops.HashAggregate(ctx, [capi.INT32], descs_of(aggs, inputs))
    sink_all(ctx, agg, keys, inputs, [0, n // 3, n])
    out = agg.finalize()
    agg.close()
    exp = reference(keys, gid, ng, inputs, aggs)
    assert (None,) in exp and exp[(7 * 1000 - 3000,)][:2] == [None, None]   # the NULL key; SUM, AVG over NULLs only
    assert_same(fetch_groups(out, 1, len(aggs)), exp, aggs, inputs)
    # every validity bit of every column, including the bits past the last group
    for c in range(out.ncols):
        _, words = raw_download(out, c)
        if out.nrows % 64:
            assert int(words[-1]) >> (out.nrows % 64) == (1 << (64 - out.nrows % 64)) - 1, (c, hex(int(words[-1])))
    out.free()


# ------------------------------------------------------------------ the 1 MiB cut
def cut_groups():
    """the largest group count whose block (INT64 key; SUM, AVG, COUNT(*) of a BIGINT) fits the host copy"""
    size = lambda g: block_bytes(g, [8, 16, 8, 8], 1)
    g = HOST_COPY_MAX // 64
    while size(g + 1) <= HOST_COPY_MAX:
        g += 1
    while size(g) > HOST_COPY_MAX:
        g -= 1
    return g


@pytest.mark.parametrize("side", ["below", "above"])
def test_cut(ctx, side):
    ng = cut_groups() + (1 if side == "above" else 0)
    rng = np.random.default_rng(5)
    gid = np.concatenate([np.arange(ng), rng.integers(0, ng, size=3 * ng)])
    key = (gid.astype(np.int64) * 7919 - 10 ** 12)
    v = rng.integers(-2 ** 63, 2 ** 63 - 1, size=len(gid), dtype=np.int64)
    valid = rng.random(len(gid)) > 0.1
    keys, inputs = [(key, None)], [(v, valid)]
    aggs = [("sum", 0), ("avg", 0), ("count_star", -1)]
    agg = ops.HashAggregate(ctx, [capi.INT64], descs_of(aggs, inputs))
    sink_all(ctx, agg, keys, inputs, [0, len(gid)])
    s0 = d2h(ctx)
    out = agg.finalize()
    s1 = d2h(ctx)
    got = fetch_groups(out, 1, len(aggs))
    s2 = d2h(ctx)
    agg.close()
    assert out.nrows == ng
    data_bytes = ng * (8 + 16 + 8 + 8) + 4 * 8 * ((ng + 63) // 64)
    if side == "below":
        assert s1 - s0 == block_bytes(ng, [8, 16, 8, 8], 1) and s2 == s1, (s0, s1, s2)
    else:
        assert s2 - s1 == data_bytes, (s0, s1, s2)   # downloads go to the device
    assert_same(got, reference(keys, gid, ng, inputs, aggs), aggs, inputs)
    out.free()


# ------------------------------------------------------------------ host-copy edge cases
def small_result(ctx, seed=3):
    rng = np.random.default_rng(seed)
    n = 50_000
    gid = rng.integers(0, 6, size=n)
    key = (gid * 3 + 1).astype(np.int16)
    v = rng.integers(-10 ** 12, 10 ** 12, size=n, dtype=np.int64)
    valid = rng.random(n) > 0.2
    keys, inputs = [(key, None)], [(v, valid)]
    aggs = [("avg", 0), ("sum", 0), ("count_star", -1), ("avg", 0)]
    agg = ops.HashAggregate(ctx, [capi.INT16], descs_of(aggs, inputs))
    sink_all(ctx, agg, keys, inputs, [0, n])
    return agg, reference(keys, gid, 6, inputs, aggs), aggs, inputs


def test_download_after_destroy(ctx):
    agg, exp, aggs, inputs = small_result(ctx)
    out = agg.finalize()
    agg.close()
    assert_same(fetch_groups(out, 1, len(aggs)), exp, aggs, inputs)
    out.free()


def test_free_without_download(ctx):
    for seed in (1, 2, 3):   # the freed result's pinned copy goes back to the cache and serves the next one
        agg, exp, aggs, inputs = small_result(ctx, seed)
        agg.finalize().free()
        out = agg.finalize()
        agg.close()
        assert_same(fetch_groups(out, 1, len(aggs)), exp, aggs, inputs)
        out.free()


def test_zero_groups(ctx):
    for sink_empty in (False, True):
        agg = ops.HashAggregate(ctx, [capi.INT64, capi.UINT8],
                                [(capi.AGG_AVG, capi.INT64, 0), (capi.AGG_SUM, capi.INT64, 0),
                                 (capi.AGG_COUNT_STAR, capi.INT64, -1)])
        if sink_empty:
            e = np.zeros(0, dtype=np.int64)
            agg.sink(ops.Batch.upload(ctx, [ops.Vector.flat(e), ops.Vector.flat(e.astype(np.uint8)),
                                            ops.Vector.flat(e)], 0), [0, 1], [2])
        out = agg.finalize()
        agg.close()
        assert out.nrows == 0 and out.ncols == 5
        res = out.download_all()
        assert all(len(v) == 0 and len(ok) == 0 for v, ok in res)
        out.free()


def test_device_view_matches_download(ctx):
    agg, exp, aggs, inputs = small_result(ctx)
    out = agg.finalize()
    agg.close()
    n = out.nrows
    for c in range(out.ncols):
        info = out.column_info(c)
        data, words = raw_download(out, c)
        assert np.array_equal(device_bytes(info.data, len(data)), data), c   # AVG columns included
        dev_words = device_bytes(info.validity, 8 * len(words)).view(np.uint64)
        assert np.array_equal(dev_words, words), c
    assert_same(fetch_groups(out, 1, len(aggs)), exp, aggs, inputs)
    assert n == 6
    out.free()
