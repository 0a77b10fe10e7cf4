"""Time filtered aggregates (b200_agg_create_filtered) on the TPC-H Q1 shape at SF100: 592 M rows, keys
(l_returnflag, l_linestatus) as u8 x u8 (bench_data.py's Q1 columns, 4 groups), four SUMs over qty, price, disc_price
and charge.  Three arms on the same device-resident columns:

  (a) the 4 SUMs unfiltered;
  (b) the same 4 SUMs, SUM j filtered by its own BOOL column f_j, the shape DuckDB binds a 4-value PIVOT to
      (f_j = pv == j for a pivot column pv in 0..3: every row passes exactly one filter);
  (c) the 4 SUMs with no filter over inputs whose validity masks are f_j: the nullable sink path without the fold,
      so (b) - (c) is the fold's cost and (c) - (a) that of the nullable sink path.

A step creates the aggregate, sinks the whole batch in one call and finalizes (the result comes back to the host).
Steps are timed with CUDA events on the context's stream, the arms alternating step by step; the median is reported.
The fold kernel's own time comes from one separate step of (b) under torch.profiler.  Its algorithmic bytes are 1 B per
row for each filter column read, plus 1/8 B per row of input validity read (the inputs here carry none), plus 1/8 B per
row of validity written, per filtered pair; the share of the H100 SXM data sheet's 3.35 TB/s is reported from them.
Every arm's result is checked against exact per-group integer sums (per-chunk int64 sums accumulated in Python ints).

    python scripts/agg_filter_bench.py [--rows 592000000] [--steps 10] [--warmup 2]
prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
SUMS = ["qty", "price", "disc_price", "charge"]


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


def pack_validity(torch, mask):
    """bool tensor -> DuckDB validity words (int64 tensor, bit i of word i // 64 = row i)"""
    n = mask.numel()
    pad = (-n) % 64
    bits = torch.cat([mask, torch.zeros(pad, dtype=torch.bool, device=mask.device)]) if pad else mask
    weights = (1 << torch.arange(8, device=mask.device, dtype=torch.int32)).to(torch.uint8)
    packed = (bits.view(-1, 8).to(torch.uint8) * weights).sum(dim=1, dtype=torch.int32).to(torch.uint8)
    return packed.view(torch.int64).contiguous()


def exact_sums(torch, cols, gid, masks, chunk=1 << 24):
    """{(group, j): sum of SUMS[j] over the group's rows (where masks[j], when given)} as Python ints"""
    out = {}
    for lo in range(0, gid.numel(), chunk):
        hi = min(gid.numel(), lo + chunk)
        g = gid[lo:hi]
        for j, name in enumerate(SUMS):
            v = cols[name][lo:hi]
            if masks is not None:
                v = torch.where(masks[j][lo:hi], v, torch.zeros_like(v))
            part = torch.zeros(4, dtype=torch.int64, device=v.device).index_add_(0, g, v).cpu().numpy()
            for k in range(4):
                out[(k, j)] = out.get((k, j), 0) + int(part[k])
    return out


def result_of(batch):
    res = batch.download_all()
    return {(int(res[0][0][g]), int(res[1][0][g])): [res[2 + j][0][g] if res[2 + j][1][g] else None
                                                      for j in range(len(SUMS))] for g in range(batch.nrows)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=592_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench_data import Gen, hmod
    from duckdb_b200 import capi
    from duckdb_b200 import operators as ops

    if not torch.cuda.is_available():
        sys.exit("agg_filter_bench.py measures on a CUDA device; there is none")
    torch.cuda.set_device(0)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    n = args.rows
    cols = Gen(torch, "cuda:0").q1(n)
    pv = Gen(torch, "cuda:0")._fill(n, 0, [("pv", torch.int8, lambda i, c: hmod(i, 23, 4))])["pv"]
    filt = [pv == j for j in range(4)]
    del pv
    valid = [pack_validity(torch, f) for f in filt]
    combo = {(82, 70): 0, (78, 70): 1, (78, 79): 2, (65, 70): 3}
    gid = ((cols["rf"] == 78).long() + ((cols["rf"] == 78) & (cols["ls"] == 79)).long() +
           3 * (cols["rf"] == 65).long())
    torch.cuda.synchronize()
    exact = {"a": exact_sums(torch, cols, gid, None), "b": exact_sums(torch, cols, gid, filt)}
    exact["c"] = exact["b"]
    del gid

    keys = [(cols["rf"].data_ptr(), capi.UINT8), (cols["ls"].data_ptr(), capi.UINT8)]
    plain = [(cols[c].data_ptr(), capi.INT64) for c in SUMS]
    arms = {
        "a": (keys + plain, None),
        "b": (keys + plain + [(f.data_ptr(), capi.BOOL) for f in filt], [4, 5, 6, 7]),
        "c": (keys + [(cols[c].data_ptr(), capi.INT64, valid[j].data_ptr()) for j, c in enumerate(SUMS)], None),
    }
    batches = {a: ops.Batch.wrap(ctx, c, n) for a, (c, _) in arms.items()}
    descs = [(capi.AGG_SUM, capi.INT64, j) for j in range(len(SUMS))]

    def step(arm):
        _, filters = arms[arm]
        agg = ops.HashAggregate(ctx, [capi.UINT8, capi.UINT8], descs, filters=filters)
        agg.sink(batches[arm], [0, 1], list(range(2, batches[arm].ncols)))
        out = agg.finalize()
        agg.close()
        return out

    checked = {}
    for arm in arms:
        got = result_of(step(arm))
        want = {k: [exact[arm][(g, j)] for j in range(len(SUMS))] for k, g in combo.items()}
        checked[arm] = got == want
        assert got == want, (arm, got, want)

    stream = torch.cuda.current_stream()
    times = {a: [] for a in arms}
    for s in range(args.warmup + args.steps):
        for arm in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            out = step(arm)
            e1.record(stream)
            e1.synchronize()
            out.free()
            if s >= args.warmup:
                times[arm].append(e0.elapsed_time(e1))

    # the fold's own time, and the kernels of one filtered step
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.02)   # idle margins keep the step inside the profiler's window (tests/kernel_trace.py)
        step("b").free()
        torch.cuda.synchronize()
        time.sleep(0.02)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    kernels = {}
    for e in events:
        if e.get("cat") == "kernel":
            name = e["name"].split("(")[0].replace("void ", "")
            kernels[name] = kernels.get(name, 0.0) + e.get("dur", 0) / 1e3   # us -> ms
    fold_ms = sum(v for k, v in kernels.items() if "agg_filter_fold_kernel" in k)
    fold_bytes = n * len(SUMS) * (1 + 1 / 8)
    med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
    res = {"workload": "agg_filter_q1_sf100", "rows": n, "sums": SUMS, **gpu_identity(),
           "arms": {a: {"ms": spread(times[a]), "rows_per_s_median": n / (med[a] / 1e3), "same_result": checked[a]}
                    for a in arms},
           "b_over_a_median": med["b"] / med["a"], "c_over_a_median": med["c"] / med["a"],
           "fold_kernel_ms": fold_ms, "fold_algorithmic_bytes": fold_bytes, "fold_input_validity_bytes": 0,
           "fold_hbm_fraction": fold_bytes / (fold_ms / 1e3) / HBM_PEAK if fold_ms else None,
           "hbm_peak_bytes_per_s": HBM_PEAK,
           "filtered_step_kernels_ms": {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])[:8]}}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
