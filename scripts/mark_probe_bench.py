"""Time the in-order MARK probe (b200_join_probe_mark) against the MARK path of b200_join_probe on the TPC-H Q14 key
sets: build = part's 20 M keys 1 .. 20 M (SF100), probe = 600 M l_partkey values (bench_data.py's formula, every row
matches).  Both calls run on the same device-resident batch; the old path writes a mark column through the generic
probe's output cursor and returns its count to the host, the new one writes every row's mark in place.

Algorithmic bytes of the new kernel: the 8-byte key read, the 1-byte mark and 1/8 byte of validity written per row;
the table's random reads are not counted (the dense table is 80 MB, larger than the H100's 50 MB L2).  Share of
peak = those bytes over the kernel time, against the 3.35 TB/s of the H100 SXM data sheet.  Each step is timed with
CUDA events on the context's stream; the two paths alternate step by step, and the marks of both are compared once
(the old path's, put back in probe order by its lhs_sel) before timing.

    python scripts/mark_probe_bench.py [--rows 600000000] [--build-rows 20000000] [--steps 10] [--warmup 2]
                                       [--tables dense,hash]
prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def gpu_identity():
    import torch
    ident = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        ident["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        ident["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return ident


def spread(ms):
    s = sorted(ms)
    return {"min": s[0], "median": s[len(s) // 2], "max": s[-1], "steps": ms}


def run_table(ctx, probe_keys, build_keys, no_dense, steps, warmup):
    import torch
    from duckdb_b200 import capi
    from duckdb_b200 import operators as ops

    n, nb = probe_keys.numel(), build_keys.numel()
    if no_dense:
        os.environ["B200_JOIN_NO_DENSE"] = "1"
    else:
        os.environ.pop("B200_JOIN_NO_DENSE", None)
    j = ops.HashJoin(ctx, capi.JOIN_MARK, [capi.INT64], [])
    j.sink(ops.Batch.wrap(ctx, [(build_keys.data_ptr(), capi.INT64)], nb), [0], [])
    j.finalize()
    os.environ.pop("B200_JOIN_NO_DENSE", None)
    probe = ops.Batch.wrap(ctx, [(probe_keys.data_ptr(), capi.INT64)], n)
    mark = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    valid = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda:0")

    def new():
        j.probe_mark(probe, [0], mark.data_ptr(), valid.data_ptr())

    def old(sel=None):
        out, count = j.execute(probe, [0], [], n, sel.data_ptr() if sel is not None else None)
        return out, count

    # same marks and validity: the old path's result rows put back in probe order by its lhs_sel
    new()
    sel = torch.empty(n, dtype=torch.int32, device="cuda:0")
    out, count = old(sel)
    assert count == n, count
    old_mark, old_valid = out.download(0)
    out.free()
    order = sel.cpu().numpy()
    del sel
    new_mark = mark.cpu().numpy()
    new_valid = np.unpackbits(valid.cpu().numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
    assert np.array_equal(new_mark[order], old_mark.view(np.uint8)), "marks differ from b200_join_probe(MARK)"
    assert np.array_equal(new_valid[order], old_valid), "mark validity differs from b200_join_probe(MARK)"
    del order, new_mark, new_valid, old_mark, old_valid

    stream = torch.cuda.current_stream()
    times = {"probe_mark": [], "probe_mark_old_path": []}
    for step in range(warmup + steps):
        for name, fn in (("probe_mark", new), ("probe_mark_old_path", old)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            res = fn()
            b.record(stream)
            b.synchronize()
            if res is not None:
                res[0].free()
            if step >= warmup:
                times[name].append(a.elapsed_time(b))
    j.close()
    bytes_per_row = 8 + 1 + 1 / 8
    result = {}
    for name, ms in times.items():
        med = sorted(ms)[len(ms) // 2]
        result[name] = {"ms": spread(ms), "rows_per_s_median": n / (med / 1e3),
                        "hbm_fraction_median": n * bytes_per_row / (med / 1e3) / HBM_PEAK}
    result["speedup_median"] = result["probe_mark_old_path"]["ms"]["median"] / result["probe_mark"]["ms"]["median"]
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

    if not torch.cuda.is_available():
        sys.exit("mark_probe_bench.py measures on a CUDA device; there is none")
    torch.cuda.set_device(0)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    gen = Gen(torch, "cuda:0")
    nb = args.build_rows
    build_keys = gen.part(nb)["partkey"]
    probe_keys = gen._fill(args.rows, 0, [("partkey", torch.int64, lambda i, c: 1 + hmod(i, 19, nb))])["partkey"]
    torch.cuda.synchronize()
    res = {"workload": "mark_probe", "rows": args.rows, "build_rows": nb, "bytes_per_row": 8 + 1 + 1 / 8,
           "hbm_peak_bytes_per_s": HBM_PEAK, **gpu_identity()}
    for table in args.tables.split(","):
        res[table] = run_table(ctx, probe_keys, build_keys, table == "hash", args.steps, args.warmup)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
