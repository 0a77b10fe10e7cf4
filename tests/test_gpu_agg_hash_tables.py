"""The two aggregate hash tables under forced hash collisions, and high-cardinality sums past 2^95.

Random keys at load <= 0.69 give short probe sequences: they almost never put two live keys on one full hash, a cluster
across the last slot, or many threads inserting different keys into one cluster at once.  Here the keys are placed:

* generic table (agg.cu, `agg_find_or_create`): slot = DuckDB hash & mask, tag = (hash & ~2^63) | 1.  `murmur64_inverse`
  puts a BIGINT key on any hash; `combine_hash_preimage` gives different (BIGINT, BIGINT[, BIGINT]) tuples one full hash.
* high-cardinality (HC) table (agg_hc.cu): slot = hc_hash_words(packed key words) & mask, restated and inverted below.
  Packed words: INTEGER key -> one word (value in bytes 0..3, NULL flags in byte 4); BIGINT -> two (word 1 holds the
  flags); two BIGINTs -> three.  For three words any (k0, k1) with equal k0 ^ k1 * C1 share the full HC hash.

Every case checks keys (as a set, no duplicate group), COUNT / COUNT(*) and SUM as Python ints, SUM_NO_OVERFLOW
wrapped to int64 and AVG through ld_avg against exact references, and asserts through the kernel trace which table and
kernel ran (a fall-back computes the same answer).  The large-sum cases hold an HC table's invariant: its 64-bit words
keep at most one table lifetime (2^32 rows) of a group's sum, everything beyond stays in the generic table's 128 bits."""
import functools
import os
import re

import numpy as np
import pytest

from duckdb_b200 import capi
from duckdb_b200 import operators as ops
from kernel_trace import assert_not_ran, assert_ran, kernel_trace
from oracle.port import NULL_HASH, combine_hash_preimage, hash_columns, murmur64, murmur64_inverse
from test_gpu_agg_kernel_paths import exact_group_sums, ld_avg, traced_window
from test_gpu_kernel_paths import _download_raw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
PROBE = 1 << 18          # rows of the adaptation probe chunk (b200_agg_sink)
HC_CAP = 1 << 20         # slots of a new HC table (HC_MIN_CAP) while the probe saw fewer than 2^18 groups
FUNC = {"count_star": capi.AGG_COUNT_STAR, "count": capi.AGG_COUNT, "sum": capi.AGG_SUM,
        "sum_no_overflow": capi.AGG_SUM_NO_OVERFLOW, "min": capi.AGG_MIN, "avg": capi.AGG_AVG}
# SUM, SUM_NO_OVERFLOW, AVG, COUNT of an INT64 input; SUM and AVG of a UBIGINT input; COUNT(*)
HC_AGGS = [("sum", 0), ("sum_no_overflow", 0), ("avg", 0), ("count", 0), ("sum", 1), ("avg", 1), ("count_star", -1)]

# ------------------------------------------------------------------ the HC slot hash, restated
HC_C1, HC_C2, HC_M = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0xD6E8FEB86659FD93
HC_SHIFTS = (32, 29)
HC_M_INV = pow(HC_M, -1, 1 << 64)


def hc_mix(x):
    x = (x * HC_M) & M64
    x ^= x >> HC_SHIFTS[0]
    x = (x * HC_M) & M64
    return x ^ (x >> HC_SHIFTS[1])


def hc_hash_words(k0, k1=0, k2=0, kw=1):
    """hc_hash_words of agg_hc.cu on Python ints"""
    x = k0 & M64
    if kw >= 2:
        x ^= (k1 * HC_C1) & M64
    if kw >= 3:
        x ^= (k2 * HC_C2) & M64
    return hc_mix(x)


def _unxorshift(y, s):
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x


def hc_unmix(h):
    """the word x0 = k0 ^ k1 * C1 ^ k2 * C2 whose HC hash is h"""
    x = _unxorshift(h & M64, HC_SHIFTS[1])
    x = (x * HC_M_INV) & M64
    x ^= x >> HC_SHIFTS[0]
    return (x * HC_M_INV) & M64


def hc_mix_np(x):
    """hc_mix on a uint64 array (wrapping multiplies)"""
    with np.errstate(over="ignore"):
        x = x * np.uint64(HC_M)
        x ^= x >> np.uint64(HC_SHIFTS[0])
        x = x * np.uint64(HC_M)
        return x ^ (x >> np.uint64(HC_SHIFTS[1]))


def s64(u):
    return (u & M64) - (1 << 64) if u & (1 << 63) else u & M64


def test_hc_hash_restatement_matches_the_kernel():
    """CPU: the constants and shifts of hc_hash_words in agg_hc.cu are the ones restated here, and hc_unmix inverts it.
    Without this pin a change of the kernel's hash would silently turn every forced HC case into random keys."""
    with open(os.path.join(ROOT, "duckdb_b200", "csrc", "agg_hc.cu")) as f:
        src = f.read()
    m = re.search(r"uint64_t hc_hash_words\(uint64_t k0, uint64_t k1, uint64_t k2, int KW\) \{(.*?)\n\}", src, re.S)
    assert m, "hc_hash_words not found in agg_hc.cu"
    body = re.sub(r"\s+", " ", m.group(1)).strip()
    consts = [int(c, 16) for c in re.findall(r"0x([0-9a-fA-F]+)ULL", body)]
    assert consts == [HC_C1, HC_C2, HC_M, HC_M], body
    assert [int(s) for s in re.findall(r">> (\d+)", body)] == list(HC_SHIFTS), body
    expect = ("uint64_t x = k0; if (KW >= 2) { x ^= k1 * 0x9e3779b97f4a7c15ULL; } if (KW >= 3) { x ^= k2 * "
              "0xc2b2ae3d27d4eb4fULL; } x *= 0xd6e8feb86659fd93ULL; x ^= x >> 32; x *= 0xd6e8feb86659fd93ULL; "
              "return x ^ (x >> 29);")
    assert body == expect, body
    rng = np.random.default_rng(0)
    for x in [0, 1, M64, 1 << 63] + [int(v) for v in rng.integers(0, 2 ** 63, size=200, dtype=np.int64)]:
        assert hc_unmix(hc_mix(x)) == x
        assert hc_mix(hc_unmix(x)) == x
    xs = rng.integers(0, 2 ** 63, size=100, dtype=np.int64).astype(np.uint64)
    assert [int(v) for v in hc_mix_np(xs)] == [hc_mix(int(v)) for v in xs]
    k0, k1 = 12345, -77 & M64
    assert hc_hash_words(k0 ^ ((k1 * HC_C1) & M64) ^ ((5 * HC_C1) & M64), 5, 0, 3) == hc_hash_words(k0, k1, 0, 3)


# ------------------------------------------------------------------ the cases run in a child process
def _serve(pipe):
    """the child process of child(): one context, runs the named cases of this module until it receives None"""
    import traceback

    import torch

    torch.cuda.set_device(0)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    pipe.send(True)
    while True:
        request = pipe.recv()
        if request is None:
            break
        name, args, env = request
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            globals()[name](ctx, *args)
            pipe.send(("ok", None))
        except Exception as e:  # a failed assertion fails the test that sent the case
            pipe.send(("assert" if isinstance(e, AssertionError) else "error", traceback.format_exc()))
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    ctx.close()
    pipe.close()


@pytest.fixture(scope="module")
def child():
    """a pipe to the child process that runs this module's GPU cases.  The large cases (multi-GB batches, 6 * 10^9
    rows) run there so that whatever they leave in a process (its memory pools, its CUPTI activity tracing, which the
    kernel-path tests of later modules rely on) ends with the child when the module is done."""
    import multiprocessing

    spawn = multiprocessing.get_context("spawn")
    parent, conn = spawn.Pipe()
    proc = spawn.Process(target=_serve, args=(conn,), daemon=True)
    proc.start()
    conn.close()
    try:
        assert parent.recv()
        yield parent
        parent.send(None)
        proc.join(timeout=120)
    finally:
        if proc.is_alive():
            proc.terminate()
            proc.join()
        parent.close()


def run_case(pipe, name, *args, env=None):
    """run case `name`(ctx, *args) in the child with the environment variables `env` set"""
    pipe.send((name, args, env or {}))
    status, result = pipe.recv()
    if status != "ok":
        raise (AssertionError if status == "assert" else RuntimeError)(result)


# ------------------------------------------------------------------ exact checks
def agg_descs(aggs, in_types):
    return [(FUNC[f], in_types[i] if i >= 0 else capi.INT64, i) for f, i in aggs]


def expected_states(gid, ng, inputs):
    """-> rows per group, [(cnt, exact sum) per input]"""
    rows = np.bincount(gid, minlength=ng).astype(np.int64)
    st = []
    for v, valid in inputs:
        cnt = rows if valid is None else np.bincount(gid, weights=valid, minlength=ng).astype(np.int64)
        st.append((cnt.astype(object), exact_group_sums(gid, ng, v, valid)))
    return rows.astype(object), st


def check_result(res, out_g, present, rows, st, aggs, in_types, mins=None):
    """finalize()'s raw columns against the exact per-group states; out_g: the group of every output row"""
    out_g = np.asarray(out_g, dtype=np.int64)
    assert len(np.unique(out_g)) == len(out_g), "duplicate group in the output"
    assert set(out_g.tolist()) == set(np.asarray(present).tolist()), "the output's groups differ from the input's"
    nk = len(res) - len(aggs)
    for a, (f, i) in enumerate(aggs):
        v, ok = res[nk + a]
        r = rows[out_g]
        if f == "count_star":
            assert (v.view(np.int64).astype(object) == r).all(), "COUNT(*) differs"
            continue
        cnt, s = st[i][0][out_g], st[i][1][out_g]
        has = cnt > 0
        if f == "count":
            assert (v.view(np.int64).astype(object) == cnt).all(), f"COUNT of input {i} differs"
            continue
        np.testing.assert_array_equal(ok, has.astype(bool))
        has = has.astype(bool)
        if f == "sum":
            bad = np.nonzero(v[has] != s[has])[0]
            assert len(bad) == 0, (f"SUM of input {i} differs", [(v[has][b], s[has][b]) for b in bad[:5]])
        elif f == "sum_no_overflow":
            wrapped = np.array([(int(x) + 2 ** 63) % 2 ** 64 - 2 ** 63 for x in s[has]], dtype=np.int64)
            np.testing.assert_array_equal(v.view(np.int64)[has], wrapped)
        elif f == "avg":
            exp = np.array([ld_avg(int(x), int(c)) for x, c in zip(s[has], cnt[has])], dtype=np.float64)
            np.testing.assert_array_equal(v[has], exp)
        elif f == "min":
            np.testing.assert_array_equal(v[has].astype(np.int64), mins[out_g][has])
        else:
            raise ValueError(f)


def group_of_keys(res, nk, key_table):
    """output rows -> group ids, through {key tuple: group}; NULL keys as None"""
    cols = [(res[j][0].tolist(), res[j][1].tolist()) for j in range(nk)]
    out = []
    for r in range(len(cols[0][0])):
        k = tuple(int(c[0][r]) if c[1][r] else None for c in cols)
        assert k in key_table, f"the output holds a key {k} no input row has"
        out.append(key_table[k])
    return out


def input_pair(rng, n):
    """an INT64 column over the full range and a UBIGINT column, with the extremes planted"""
    x = rng.integers(-2 ** 63, 2 ** 63, size=n, dtype=np.int64)
    y = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    for v, edges in ((x, [-2 ** 63, 2 ** 63 - 1]), (y, [2 ** 64 - 1, 2 ** 63])):
        for e in edges:
            v[rng.integers(0, n, size=200)] = e
    return x, y


def race_order(rng, clustered, background, n_probe, n_tail):
    """row -> group: n_probe background rows (the adaptation probe sees them all), then every clustered group in 64
    adjacent rows (many threads race to insert the keys of one cluster), then n_tail rows of both, shuffled"""
    probe = rng.choice(background, size=n_probe)
    race = np.repeat(clustered, 64)
    tail = rng.choice(np.concatenate([clustered, background]), size=n_tail)
    return np.concatenate([probe, race, tail]).astype(np.int64)


# ------------------------------------------------------------------ generic table (agg.cu)
GENERIC_AGGS = [("sum", 0), ("sum_no_overflow", 0), ("avg", 0), ("count", 0), ("min", 0), ("sum", 1),
                ("count_star", -1)]
GENERIC_VARIANTS = ["fullhash64", "fullhash1024", "tag_alias", "null_hash", "growth", "combine"]
LAST = 0xFFFFFFFF  # a hash whose low 32 bits are all ones is homed on the last slot of every table up to 2^32 slots


def tuples_on_hash(rng, target, count):
    """`count` distinct (BIGINT, BIGINT) tuples whose DuckDB hash, combine(murmur64(k0), murmur64(k1)), is `target`"""
    out = set()
    while len(out) < count:
        k0 = int(rng.integers(-2 ** 63, 2 ** 63, dtype=np.int64))
        k1 = combine_hash_preimage(int(murmur64(np.uint64(k0 & M64))), target)
        out.add((k0, s64(k1)))
    out = sorted(out)
    h = hash_columns([(np.array([k[j] for k in out], dtype=np.int64), None) for j in range(2)])
    assert (h == np.uint64(target)).all()
    return out


def generic_case(variant, seed):
    """-> (key columns [(values, valid)], group key table, gid, ng, what the case is about)"""
    rng = np.random.default_rng(seed)
    if variant == "null_hash":
        # one BIGINT key whose hash is NULL_HASH, NULL keys, 1000 ordinary keys: two groups, not one
        special = s64(murmur64_inverse(int(NULL_HASH)))
        assert int(murmur64(np.uint64(special & M64))) == int(NULL_HASH)
        ordinary = rng.integers(-2 ** 62, 2 ** 62, size=1000, dtype=np.int64)
        keys = [(special,), (None,)] + [(int(k),) for k in ordinary]
        clustered = np.arange(2)
    else:
        targets = {"fullhash64": [(0x5A5A << 48) | LAST],
                   "fullhash1024": [(0x1234 << 48) | LAST],
                   "tag_alias": [t for t0 in [(0x0F0F << 48) | (LAST - 1)] for t in
                                 (t0, t0 ^ 1, t0 ^ (1 << 63), t0 ^ 1 ^ (1 << 63))],
                   "growth": [(0x77 << 56) | (LAST - 3 * i) for i in range(4)],
                   "combine": [(0x4242 << 48) | LAST, (0x2424 << 48) | (LAST - 64)]}[variant]
        per = {"fullhash64": 64, "fullhash1024": 1024, "tag_alias": 64, "growth": 1024, "combine": 512}[variant]
        keys = [k for t in targets for k in tuples_on_hash(rng, t, per)]
        nord = 40_000 if variant == "growth" else 1000
        keys += [tuple(int(v) for v in r) for r in rng.integers(-2 ** 62, 2 ** 62, size=(nord, 2), dtype=np.int64)]
        clustered = np.arange(len(targets) * per)
    assert len(set(keys)) == len(keys)
    ng = len(keys)
    background = np.arange(len(clustered), ng)
    gid = race_order(rng, clustered, background, 20_000, 300_000)   # (more rows than the probe)
    nk = len(keys[0])
    cols = []
    for j in range(nk):
        vals = np.array([0 if k[j] is None else k[j] for k in keys], dtype=np.int64)
        valid = np.array([k[j] is not None for k in keys])
        cols.append((vals[gid], None if valid.all() else valid[gid]))
    return cols, {k: g for g, k in enumerate(keys)}, gid, ng


@pytest.mark.gpu
@pytest.mark.parametrize("variant", GENERIC_VARIANTS)
def test_generic_table_forced_collisions(child, variant):
    run_case(child, "generic_table_case", variant)


def generic_table_case(ctx, variant):
    """Keys forced onto one full hash (64 and 1024 BIGINT pairs), onto four hashes that share one tag (bits 0 and 63),
    onto NULL_HASH next to NULL keys, homed on the last slot so probing wraps to slot 0, clusters that make the sink
    cross the exact fill limit (defer, rehash from the stored hash, replay), and clustered partial tables through
    export_states -> combine_states.  MIN keeps the rows out of the HC table; every clustered key first arrives in 64
    adjacent rows."""
    cols, key_table, gid, ng = generic_case(variant, seed=GENERIC_VARIANTS.index(variant))
    n = len(gid)
    rng = np.random.default_rng(5)
    x, y = input_pair(rng, n)
    inputs = [(x, None), (y, None)]
    in_types = [capi.INT64, capi.UINT64]
    key_types = [capi.INT64] * len(cols)
    descs = agg_descs(GENERIC_AGGS, in_types)

    def sink(a, lo, hi):
        vs = [ops.Vector.flat(k[lo:hi], None if kv is None else kv[lo:hi]) for k, kv in cols]
        vs += [ops.Vector.flat(x[lo:hi]), ops.Vector.flat(y[lo:hi])]
        a.sink(ops.Batch.upload(ctx, vs, hi - lo), list(range(len(cols))), [len(cols), len(cols) + 1])

    def run():
        if variant == "combine":
            parts = []
            for lo, hi in ((0, n // 2), (n // 2, n)):
                a = ops.HashAggregate(ctx, key_types, descs)
                sink(a, lo, hi)
                parts.append(a)
            agg = ops.HashAggregate(ctx, key_types, descs)
            for a in parts:
                agg.combine_states(a.export_states())
                a.close()
        else:
            agg = ops.HashAggregate(ctx, key_types, descs)
            sink(agg, 0, n)
        out = _download_raw(agg.finalize())
        agg.close()
        return out

    res, names = traced_window(run, always=["agg_init_kernel"])
    rows, st = expected_states(gid, ng, inputs)
    mins = np.full(ng, 2 ** 63 - 1, dtype=np.int64)
    np.minimum.at(mins, gid, x)
    out_g = group_of_keys(res, len(cols), key_table)
    check_result(res, out_g, np.unique(gid), rows, st, GENERIC_AGGS, in_types, mins=mins)
    assert_ran(names, "agg_sink_kernel", "agg_finalize_kernel")
    assert_not_ran(names, "agg_hc_direct_kernel", "agg_hc_simple_kernel", "agg_hc_kernel", "agg_hc_rows_kernel")
    if variant == "growth":
        assert_ran(names, "agg_rehash_kernel")
    if variant == "combine":
        assert_ran(names, "agg_export_kernel", "agg_combine_kernel")


# ------------------------------------------------------------------ HC table (agg_hc.cu)
WINDOWS = (HC_CAP - 64, 123_456)   # 64-slot windows: one ends at the last slot of the table
WINDOW_KEYS = (2048, 1024)


@functools.lru_cache(maxsize=None)
def int32_window_keys():
    """INTEGER keys whose HC slot in a 2^20-slot table falls in each window: a bounded brute force over 4 * 10^7
    candidates (about 2400 per window)"""
    found = [[], []]
    step = 1 << 23
    for lo in range(0, 40_000_000, step):
        v = np.arange(lo, min(lo + step, 40_000_000), dtype=np.uint64)
        slot = hc_mix_np(v) & np.uint64(HC_CAP - 1)
        for w, start in enumerate(WINDOWS):
            found[w].append(v[(slot >= np.uint64(start)) & (slot < np.uint64(start + 64))])
    out = []
    for w in range(2):
        keys = np.concatenate(found[w])[:WINDOW_KEYS[w]]
        assert len(keys) == WINDOW_KEYS[w], "the brute force found too few keys for a window"
        out.append(keys.astype(np.int64))
    return out


def hc_window_hash(rng, w, j):
    """a full HC hash homed on slot j of window w in every table of 2^20 .. 2^26 slots"""
    return (int(rng.integers(0, 2 ** 38)) << 26) | (WINDOWS[w] + j % 64)


def hc_case_keys(kw, rng, nbg):
    """-> key tuples (clustered first), count of clustered keys.  kw 3: groups of 16 keys share one full hash."""
    keys = []
    if kw == 1:
        for w in range(2):
            keys += [(int(k),) for k in int32_window_keys()[w]]
        bg = -(np.arange(1, nbg + 1, dtype=np.int64) * 7)          # negative: disjoint from the brute-forced keys
        ncl = len(keys)
        keys += [(int(k),) for k in bg]
        return keys, ncl
    for w in range(2):
        for j in range(WINDOW_KEYS[w] if kw == 2 else WINDOW_KEYS[w] // 16):
            x0 = hc_unmix(hc_window_hash(rng, w, j))
            if kw == 2:
                keys.append((s64(x0),))
            else:
                for k1 in rng.integers(-2 ** 63, 2 ** 63, size=16, dtype=np.int64):
                    k1 = int(k1) & M64
                    keys.append((s64(x0 ^ ((k1 * HC_C1) & M64)), s64(k1)))
    ncl = len(keys)
    bg = rng.integers(-2 ** 63, 2 ** 63, size=(nbg + 100, kw - 1), dtype=np.int64)
    seen = set(keys)
    for r in bg:
        t = tuple(int(v) for v in r)
        if t not in seen:
            seen.add(t)
            keys.append(t)
        if len(keys) == ncl + nbg:
            break
    return keys, ncl


def hc_slot(kw, key, mask):
    words = [k & M64 for k in key] + [0]
    if kw == 1:
        words = [key[0] & 0xFFFFFFFF]
    return hc_hash_words(*(words + [0, 0])[:3], kw=kw) & mask


HC_KERNEL = {"direct": "agg_hc_direct_kernel<{kw}, 2>", "tile": "agg_hc_simple_kernel<{kw}>",
             "generic": "agg_hc_kernel<{kw}, false>", "nullable": "agg_hc_kernel<{kw}, false>",
             "dictionary": "agg_hc_rows_kernel<{kw}>", "growth": "agg_hc_direct_kernel<{kw}, 2>"}


@pytest.mark.gpu
# (INTEGER window keys are placed for a 2^20-slot table only: the growth case takes 2- and 3-word keys)
@pytest.mark.parametrize("kw,kernel", [(kw, k) for kw in (1, 2, 3) for k in HC_KERNEL if (kw, k) != (1, "growth")])
def test_hc_table_forced_clusters(child, kw, kernel):
    env = {"tile": {"B200_HC_TILE": "1"}, "generic": {"B200_HC_GENERIC": "1"}}.get(kernel, {})
    run_case(child, "hc_cluster_case", kw, kernel, env=env)


def hc_cluster_case(ctx, kw, kernel):
    """1-, 2- and 3-word HC keys placed in two 64-slot windows (2048 and 1024 keys; one window ends at the last slot,
    so its cluster wraps to slot 0; with 3-word keys every 16 keys share one full HC hash), next to 20 K ordinary
    groups: the adaptation probe sees them and picks the HC table (absorbing its groups), then every clustered key
    arrives in 64 adjacent rows (first-insert races on one cluster).  Each sink kernel: direct (default), staged
    (B200_HC_TILE), generic (B200_HC_GENERIC, and nullable inputs), the row kernel (a dictionary key vector); growth:
    900 K more groups push the shards past their limit, so a clustered table is rehashed and deferred rows replayed."""
    rng = np.random.default_rng(kw * 100 + len(kernel))
    nbg = 900_000 if kernel == "growth" else 20_000
    keys, ncl = hc_case_keys(kw, rng, nbg)
    ng = len(keys)
    clustered, background = np.arange(ncl), np.arange(ncl, ng)
    slots = np.array([hc_slot(kw, k, HC_CAP - 1) for k in keys[:ncl]])
    starts = np.array([WINDOWS[0]] * WINDOW_KEYS[0] + [WINDOWS[1]] * WINDOW_KEYS[1])
    assert ((slots >= starts) & (slots < starts + 64)).all(), "a clustered key is not homed in its window"
    if kernel == "growth":
        # the race rows, then every background group once: the first HC chunk (1 M rows) holds more groups than the
        # shards of a 2^20-slot table allow
        gid = np.concatenate([race_order(rng, clustered, background, 0, 0), rng.permutation(background),
                              rng.choice(np.concatenate([clustered, background]), size=100_000)])
    else:
        gid = race_order(rng, clustered, background, PROBE, 200_000)
    n = len(gid)
    x, y = input_pair(rng, n)
    xv = yv = None
    if kernel == "nullable":
        xv, yv = rng.random(n) > 0.2, rng.random(n) > 0.3
    kcols = [np.array([k[j] for k in keys], dtype=np.int32 if kw == 1 else np.int64) for j in range(len(keys[0]))]
    key_types = [capi.INT32 if kw == 1 else capi.INT64] * len(kcols)
    in_types = [capi.INT64, capi.UINT64]
    descs = agg_descs(HC_AGGS, in_types)

    def run():
        agg = ops.HashAggregate(ctx, key_types, descs, expected_groups=ng if kernel == "dictionary" else 0)
        if kernel == "dictionary":
            vs = [ops.Vector.dictionary(c, gid.astype(np.uint32)) for c in kcols]
        else:
            vs = [ops.Vector.flat(c[gid]) for c in kcols]
        vs += [ops.Vector.flat(x, xv), ops.Vector.flat(y, yv)]
        agg.sink(ops.Batch.upload(ctx, vs, n), list(range(len(kcols))), [len(kcols), len(kcols) + 1])
        out = _download_raw(agg.finalize())
        agg.close()
        return out

    with kernel_trace() as names:
        res = run()
    rows, st = expected_states(gid, ng, [(x, xv), (y, yv)])
    out_g = group_of_keys(res, len(kcols), {k: g for g, k in enumerate(keys)})
    check_result(res, out_g, np.unique(gid), rows, st, HC_AGGS, in_types)
    assert_ran(names, HC_KERNEL[kernel].format(kw=kw), f"agg_hc_finalize_kernel<{kw}>")
    if kw < 3 and kernel != "dictionary":
        assert_ran(names, f"agg_hc_absorb_kernel<{kw}>")
    if kernel == "growth":
        assert_ran(names, f"agg_hc_rehash_kernel<{kw}>", f"agg_hc_rows_kernel<{kw}>", "hc_spread_count_kernel")
    assert_not_ran(names, "agg_hc_flush_kernel")       # (finalize reads the HC table)
    if kw == 3:
        assert_not_ran(names, "agg_sink_kernel")       # (3-word keys go to the HC table from the first row)


# ------------------------------------------------------------------ sums past 2^95
LARGE = [2 ** 100, -2 ** 100, 2 ** 95 - 2 ** 40, -(2 ** 95 - 2 ** 40)]


def large_sum_data(seed, G=5000):
    rng = np.random.default_rng(seed)
    keys = (np.arange(G, dtype=np.int64) * 1_000_003 - 2 ** 40)
    parts = []
    for n in (PROBE + (1 << 17), PROBE + (1 << 16), 1 << 17):   # partial A, then B's two sinks
        gid = rng.integers(0, G, size=n)
        x, y = input_pair(rng, n)
        parts.append((gid, x, y))
    return keys, parts


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["states", "packed"])
def test_hc_large_sums_after_combine(child, route):
    run_case(child, "large_sums_case", route)


def large_sums_case(ctx, route):
    """A partial whose sums stand for about 2^37 rows (+-2^100 and +-(2^95 - 2^40) added to chosen groups' exported
    sum words, rows / cnt raised by 2^37) is combined into an aggregate on the HC path, which then sinks more rows and
    finalizes.  The HC table made after the combine must start empty: absorbing the combined groups would keep 96 bits
    of their sums.  Exact SUM / SUM_NO_OVERFLOW / AVG of an INT64 and a UBIGINT input; export_states -> combine_states
    and export_packed -> combine_packed (one rank)."""
    import torch

    G = 5000
    keys, parts = large_sum_data(11 + len(route), G)
    in_types = [capi.INT64, capi.UINT64]
    descs = agg_descs(HC_AGGS, in_types)
    chosen = np.arange(0, 40, 5)                       # groups whose partial state is raised
    dx = {int(g): LARGE[k % 4] for k, g in enumerate(chosen)}
    dy = {int(g): abs(LARGE[k % 4]) for k, g in enumerate(chosen)}
    dr = 2 ** 37

    def batch(gid, x, y):
        return ops.Batch.upload(ctx, [ops.Vector.flat(keys[gid]), ops.Vector.flat(x), ops.Vector.flat(y)], len(gid))

    def raise_states(kcol, cols):
        """cols: [rows, cnt0, lo0, hi0, cnt1, lo1, hi1] uint64 arrays, modified in place"""
        for r, k in enumerate(kcol):
            g = int((int(k) + 2 ** 40) // 1_000_003)
            if g not in dx:
                continue
            for c in (0, 1, 4):
                cols[c][r] = np.uint64(int(cols[c][r]) + dr)
            for (lo, hi), d in (((2, 3), dx[g]), ((5, 6), dy[g])):
                s = int(cols[lo][r]) + (s64(int(cols[hi][r])) << 64) + d
                cols[lo][r], cols[hi][r] = np.uint64(s & M64), np.uint64((s >> 64) & M64)

    def run():
        a = ops.HashAggregate(ctx, [capi.INT64], descs)
        a.sink(batch(*parts[0]), [0], [1, 2])
        b = ops.HashAggregate(ctx, [capi.INT64], descs)
        b.sink(batch(*parts[1]), [0], [1, 2])
        if route == "states":
            raw = _download_raw(a.export_states())
            kcol = raw[0][0].astype(np.int64)
            cols = [raw[c][0].astype(np.uint64) for c in range(1, 8)]
            raise_states(kcol, cols)
            b.combine_states(ops.Batch.upload(ctx, [ops.Vector.flat(kcol)] + [ops.Vector.flat(c) for c in cols],
                                              len(kcol)))
        else:
            words = a.packed_words(G)
            buf = torch.zeros(words, dtype=torch.int64, device="cuda:0")
            a.export_packed(buf.data_ptr(), G)
            host = buf.cpu().numpy().view(np.uint64).copy()
            ngr = int(host[0])
            assert ngr == G and host[1] == 0
            kcol = host[2:2 + ngr].view(np.int64)
            base = 2 + 2 * G                           # one key column, the NULL-bits column, then the states
            cols = [host[base + c * G: base + c * G + ngr] for c in range(7)]   # views: modified in place
            raise_states(kcol, cols)
            buf.copy_(torch.from_numpy(host.view(np.int64)).to("cuda:0"))
            b.combine_packed(buf.data_ptr(), 1, G)
            ctx.sync()
        b.sink(batch(*parts[2]), [0], [1, 2])
        out = _download_raw(b.finalize())
        a.close()
        b.close()
        return out

    res, names = traced_window(run, always=["agg_init_kernel"])
    gid = np.concatenate([p[0] for p in parts])
    rows, st = expected_states(gid, G, [(np.concatenate([p[1] for p in parts]), None),
                                        (np.concatenate([p[2] for p in parts]), None)])
    for g in chosen:
        rows[g] += dr
        st[0][0][g] += dr
        st[1][0][g] += dr
        st[0][1][g] += dx[int(g)]
        st[1][1][g] += dy[int(g)]
    out_g = ((res[0][0].astype(np.int64) + 2 ** 40) // 1_000_003).tolist()
    check_result(res, out_g, np.arange(G), rows, st, HC_AGGS, in_types)
    assert_ran(names, "agg_hc_direct_kernel<2, 2>", "agg_hc_flush_kernel<2>",
               "agg_combine_kernel" if route == "states" else "agg_combine_packed_kernel")


@pytest.mark.gpu
def test_hc_retirement_between_batches(child):
    run_case(child, "retirement_case")


def retirement_case(ctx):
    """One device-resident batch of 2^28 rows (INTEGER keys over 2^20 groups, INT64 values -2^63 and 2^63 - 1) sunk 17
    times: after 16 sinks the HC table holds its lifetime of 2^32 rows, so the 17th batch's first chunk retires it
    into the generic table and a new, empty table takes the rest.  The answer is 17 x the per-batch states."""
    import torch

    n, G, R = 1 << 28, 1 << 20, 17
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(3)
    keys = torch.randint(0, G, (n,), dtype=torch.int32, device="cuda:0", generator=gen)
    neg = torch.randint(0, 2, (n,), dtype=torch.int64, device="cuda:0", generator=gen)
    cnt = torch.zeros(2 * G, dtype=torch.int64, device="cuda:0")
    for lo in range(0, n, 1 << 26):
        cnt += torch.bincount(keys[lo:lo + (1 << 26)].to(torch.int64) * 2 + neg[lo:lo + (1 << 26)], minlength=2 * G)
    vals = torch.full((n,), 2 ** 63 - 1, dtype=torch.int64, device="cuda:0")
    vals.masked_fill_(neg.bool(), -2 ** 63)
    del neg
    cnt = cnt.view(G, 2).cpu().numpy()
    aggs = [("sum", 0), ("sum_no_overflow", 0), ("avg", 0), ("count", 0), ("count_star", -1)]
    agg = ops.HashAggregate(ctx, [capi.INT32], agg_descs(aggs, [capi.INT64]))
    b = ops.Batch.wrap(ctx, [(keys.data_ptr(), capi.INT32), (vals.data_ptr(), capi.INT64)], n, keepalive=(keys, vals))
    with kernel_trace() as names:
        for _ in range(R):
            agg.sink(b, [0], [1])
        res = _download_raw(agg.finalize())
    agg.close()
    del b, keys, vals
    torch.cuda.empty_cache()
    pos, ng_ = cnt[:, 0].astype(object), cnt[:, 1].astype(object)
    rows = (pos + ng_) * R
    sums = (pos * (2 ** 63 - 1) - ng_ * 2 ** 63) * R
    check_result(res, res[0][0].astype(np.int64), np.nonzero(cnt.sum(axis=1))[0], rows, [(rows, sums)], aggs,
                 [capi.INT64])
    assert_ran(names, "agg_hc_direct_kernel<1, 1>", "agg_hc_flush_kernel<1>")


@pytest.mark.gpu
def test_hc_lifetime_guard_inside_a_batch(child):
    run_case(child, "lifetime_guard_case")


def lifetime_guard_case(ctx):
    """After an HC-choosing batch of fewer than 2^19 rows, two constant batches of one key: 2^31 - 2^19 rows, then
    2^32 - 1 rows, of INT64 -1 and UBIGINT 2^64 - 1.  The second batch passes the table's lifetime of 2^32 rows in its
    middle: the guard before each chunk retires the table there, so the low-half sum of that group cannot wrap.
    Closed-form answer.  (Its run time is bound by same-address atomics on one slot.)"""
    rng = np.random.default_rng(8)
    G = 5000
    n1 = PROBE + (1 << 17)
    gid = rng.integers(0, G, size=n1)
    keys = np.arange(G, dtype=np.int32) * 3 - 7000
    x, y = input_pair(rng, n1)
    in_types = [capi.INT64, capi.UINT64]
    descs = agg_descs(HC_AGGS, in_types)
    K = 1234
    big = [(1 << 31) - (1 << 19), (1 << 32) - 1]
    agg = ops.HashAggregate(ctx, [capi.INT32], descs)
    with kernel_trace() as names:
        agg.sink(ops.Batch.upload(ctx, [ops.Vector.flat(keys[gid]), ops.Vector.flat(x), ops.Vector.flat(y)], n1),
                 [0], [1, 2])
        for m in big:
            agg.sink(ops.Batch.upload(ctx, [ops.Vector.constant(keys[K], np.int32), ops.Vector.constant(-1, np.int64),
                                            ops.Vector.constant(2 ** 64 - 1, np.uint64)], m), [0], [1, 2])
        res = _download_raw(agg.finalize())
    agg.close()
    rows, st = expected_states(gid, G, [(x, None), (y, None)])
    extra = sum(big)
    rows[K] += extra
    for i, v in enumerate((-1, 2 ** 64 - 1)):
        st[i][0][K] += extra
        st[i][1][K] += extra * v
    out_g = ((res[0][0].astype(np.int64) + 7000) // 3).tolist()
    check_result(res, out_g, np.unique(gid), rows, st, HC_AGGS, in_types)
    assert_ran(names, "agg_hc_direct_kernel<1, 2>", "agg_hc_rows_kernel<1>", "agg_hc_flush_kernel<1>")
