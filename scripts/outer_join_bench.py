"""Time the RIGHT and FULL OUTER probes against the INNER probe, and the unmatched-row scan, on the TPC-H Q14 key sets:
build = part's 20 M keys 1 .. 20 M (SF100) with a 1-byte payload (Q14's shape), probe = 600 M l_partkey values
(bench_data.py's formula, every row matches).

The three joins share one device-resident probe batch.  INNER runs the lean PK-FK kernel with the payload inline in
the table; RIGHT and FULL flag every build row they emit, so they take the tile kernel with build row ids (the dense
table keeps row ids instead of inline payloads).  The scan (b200_join_scan_unmatched over every build row) runs after
the RIGHT probes; it returns the build rows no probe matched.  Every step is timed with CUDA events on the context's
stream; the calls alternate step by step.  Before timing, the three probes' row counts and the scan's count are
checked against the key sets.

    python scripts/outer_join_bench.py [--rows 600000000] [--build-rows 20000000] [--steps 10] [--warmup 2]
                                       [--tables dense,hash]
prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def run_table(ctx, probe_keys, build_keys, payload, no_dense, steps, warmup):
    import torch
    from duckdb_b200 import capi
    from duckdb_b200 import operators as ops
    from mark_probe_bench import spread

    n, nb = probe_keys.numel(), build_keys.numel()
    if no_dense:
        os.environ["B200_JOIN_NO_DENSE"] = "1"
    joins = {}
    for name, jt in (("inner", capi.JOIN_INNER), ("right", capi.JOIN_RIGHT), ("full", capi.JOIN_OUTER)):
        j = ops.HashJoin(ctx, jt, [capi.INT64], [capi.UINT8])
        j.sink(ops.Batch.wrap(ctx, [(build_keys.data_ptr(), capi.INT64), (payload.data_ptr(), capi.UINT8)], nb),
               [0], [1])
        j.finalize()
        joins[name] = j
    os.environ.pop("B200_JOIN_NO_DENSE", None)
    probe = ops.Batch.wrap(ctx, [(probe_keys.data_ptr(), capi.INT64)], n)
    matched_keys = int(torch.unique(probe_keys).numel())

    def probe_fn(name):
        out, count = joins[name].execute(probe, [0], [], n)
        out.free()
        return count

    def scan():
        out, count = joins["right"].scan_unmatched()
        out.free()
        return count

    for name in joins:
        assert probe_fn(name) == n, name              # every probe row has exactly one partner
    assert scan() == nb - matched_keys
    calls = {"inner_probe": lambda: probe_fn("inner"), "right_probe": lambda: probe_fn("right"),
             "full_probe": lambda: probe_fn("full"), "scan_unmatched": scan}
    stream = torch.cuda.current_stream()
    times = {k: [] for k in calls}
    for step in range(warmup + steps):
        for name, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            if step >= warmup:
                times[name].append(a.elapsed_time(b))
    for j in joins.values():
        j.close()
    result = {k: {"ms": spread(ms), "rows_per_s_median": (nb if k == "scan_unmatched" else n) /
                  (sorted(ms)[len(ms) // 2] / 1e3)} for k, ms in times.items()}
    inner = result["inner_probe"]["ms"]["median"]
    for k in ("right_probe", "full_probe"):
        result[k]["vs_inner_median"] = result[k]["ms"]["median"] / inner
    result["unmatched_build_rows"] = nb - matched_keys
    return result


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--build-rows", type=int, default=20_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tables", default="dense,hash", help="dense: the direct-addressed table; hash: open addressing")
    args = ap.parse_args()
    import torch
    from bench_data import Gen, hmod
    from duckdb_b200 import operators as ops
    from mark_probe_bench import gpu_identity

    if not torch.cuda.is_available():
        sys.exit("outer_join_bench.py measures on a CUDA device; there is none")
    torch.cuda.set_device(0)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    gen = Gen(torch, "cuda:0")
    nb = args.build_rows
    build_keys = gen.part(nb)["partkey"]
    payload = (build_keys % 251).to(torch.uint8)
    probe_keys = gen._fill(args.rows, 0, [("partkey", torch.int64, lambda i, c: 1 + hmod(i, 19, nb))])["partkey"]
    torch.cuda.synchronize()
    res = {"workload": "outer_join", "rows": args.rows, "build_rows": nb, **gpu_identity()}
    for table in args.tables.split(","):
        res[table] = run_table(ctx, probe_keys, build_keys, payload, table == "hash", args.steps, args.warmup)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
