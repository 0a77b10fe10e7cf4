#!/usr/bin/env python3
"""Where the time of an aggregate step goes outside the sink: the bench.py Q1 and SSB aggregates, phase by phase.

A step is HashAggregate(...) -> sink -> finalize() -> download_all() -> close(), as bench.py times it.  For each workload:
  1. host-clock phase times (create / sink / finalize / download_all / close) with a torch.cuda.synchronize() at every
     boundary, median and spread (max - min) over --steps steps after --warmup;
  2. the step time from CUDA events, steps back to back without any synchronise in between (as bench.py times them);
  3. from a separate torch.profiler run of --trace-steps steps: kernels, memcpys and memsets per step, the
     cudaStreamSynchronize / cudaEventSynchronize calls per step when the trace carries runtime-API events, and the
     GPU busy time (union of kernel, memcpy and memset intervals) against the step's host time.
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line; needs a CUDA device.

  python scripts/agg_step_profile.py [--q1-rows N] [--ssb-rows N] [--steps 20] [--warmup 5] [--out FILE]"""
import argparse
import contextlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (gpu_info, Q1_ROWS, SF100_LINEITEM: the benchmark's own shapes)
import bench_data as BD  # noqa: E402
from kernel_trace import _strip  # noqa: E402

PHASES = ("create", "sink", "finalize", "download_all", "close")


def stats(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return {"median": round(float(np.median(xs)), 4), "spread": round(float(xs.max() - xs.min()), 4),
            "min": round(float(xs.min()), 4)}


def union_us(intervals):
    total, end = 0.0, None
    for s, e in sorted(intervals):
        if end is None or s > end:
            total += e - s
            end = e
        elif e > end:
            total += e - end
            end = e
    return total


def profile_workload(torch, ops, ctx, make, sink, steps, warmup, trace_steps):
    from torch.profiler import ProfilerActivity, profile, record_function

    def step(mark=False):
        def phase(name):
            return record_function("phase:" + name) if mark else contextlib.nullcontext()

        with phase("create"):
            a = make()
        with phase("sink"):
            sink(a)
        with phase("finalize"):
            out = a.finalize()
        with phase("download_all"):
            res = out.download_all()
        with phase("close"):
            a.close()
            out.free()
        return res

    for _ in range(warmup):
        step()
    # 1. phases, synchronised at every boundary
    ph = {p: [] for p in PHASES}
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a = make()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        sink(a)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        out = a.finalize()
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        out.download_all()
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        a.close()
        out.free()
        torch.cuda.synchronize()
        t5 = time.perf_counter()
        for p, x in zip(PHASES, (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t5 - t4)):
            ph[p].append(1e3 * x)
    # 2. back-to-back steps, CUDA events (sink alone and whole step)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    sev = []
    ev[0].record()
    for i in range(steps):
        a = make()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sink(a)
        e1.record()
        sev.append((e0, e1))
        a.finalize().download_all()
        a.close()
        ev[i + 1].record()
    torch.cuda.synchronize()
    step_ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
    sink_ms = [x.elapsed_time(y) for x, y in sev]
    out = {"phases_ms": {p: stats(v) for p, v in ph.items()}, "step_ms": stats(step_ms), "sink_ms": stats(sink_ms),
           "rest_ms": stats([s - k for s, k in zip(step_ms, sink_ms)])}
    # 3. one separate profiler run
    torch.cuda.synchronize()
    s0 = ctx.stats()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(0.02)
        for _ in range(trace_steps):
            with record_function("agg_step"):
                step(mark=True)
                torch.cuda.synchronize()
        time.sleep(0.02)
    s1 = ctx.stats()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    wins = sorted((e["ts"], e["ts"] + e.get("dur", 0)) for e in events if e.get("name") == "agg_step" and "dur" in e)
    gpu = [e for e in events if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "dur" in e]
    rt = [e for e in events if e.get("cat") == "cuda_runtime"]
    per = []
    for lo, hi in wins:
        inside = [e for e in gpu if lo <= e["ts"] <= hi]
        rin = [e for e in rt if lo <= e["ts"] <= hi]
        kern = [_strip(e["name"]) for e in inside if e["cat"] == "kernel"]
        memcpy = [e["name"] for e in inside if e["cat"] == "gpu_memcpy"]
        per.append({
            "host_ms": round((hi - lo) / 1e3, 4),
            "gpu_busy_ms": round(union_us([(e["ts"], e["ts"] + e["dur"]) for e in inside]) / 1e3, 4),
            "kernels": len(kern), "kernel_names": sorted(set(kern)),
            "memcpy": len(memcpy), "memcpy_kinds": {k: memcpy.count(k) for k in sorted(set(memcpy))},
            "memset": sum(1 for e in inside if e["cat"] == "gpu_memset"),
            "stream_syncs": sum(1 for e in rin if e["name"] == "cudaStreamSynchronize") if rt else None,
            "event_syncs": sum(1 for e in rin if e["name"] == "cudaEventSynchronize") if rt else None,
        })
    # per phase (mean over the traced steps): host time, and how much of it was spent inside CUDA runtime calls
    phases = {}
    for p in PHASES:
        spans = [(e["ts"], e["ts"] + e["dur"]) for e in events if e.get("name") == "phase:" + p and "dur" in e]
        inside = [e for e in rt if "dur" in e and any(lo <= e["ts"] <= hi for lo, hi in spans)]
        calls = {}
        for e in inside:
            calls[e["name"]] = calls.get(e["name"], 0.0) + e["dur"] / 1e3 / max(1, len(spans))
        phases[p] = {"host_ms": round(sum(hi - lo for lo, hi in spans) / 1e3 / max(1, len(spans)), 4),
                     "cuda_runtime_ms": round(sum(calls.values()), 4),
                     "top_runtime_calls_ms": {k: round(v, 4) for k, v in sorted(calls.items(), key=lambda kv: -kv[1])[:4]}}
    out["trace"] = {"steps": per, "phases": phases, "runtime_events_in_trace": bool(rt),
                    "note": "each traced step ends in one torch.cuda.synchronize() of its own (not part of the step)",
                    "library_launches_per_step": (s1["launches"] - s0["launches"]) / max(1, trace_steps),
                    "library_d2h_bytes_per_step": (s1["d2h_bytes"] - s0["d2h_bytes"]) / max(1, trace_steps),
                    "library_h2d_bytes_per_step": (s1["h2d_bytes"] - s0["h2d_bytes"]) / max(1, trace_steps)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--q1-rows", type=int, default=bench.Q1_ROWS)
    ap.add_argument("--ssb-rows", type=int, default=bench.SF100_LINEITEM)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--trace-steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("agg_step_profile.py needs a CUDA device")
    from duckdb_b200 import capi
    from duckdb_b200 import operators as ops

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    gen = BD.Gen(torch, dev)
    result = {"gpu": bench.gpu_info(0)}

    # TPC-H Q1 (bench.py's headline): 2 u8 keys, 4 hugeint sums, 3 integer averages, count(*)
    q1 = gen.q1(args.q1_rows)
    cols = [q1[k] for k in ("rf", "ls", "qty", "price", "disc_price", "charge", "disc")]
    types = [capi.UINT8, capi.UINT8] + [capi.INT64] * 5
    desc = [(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_SUM, capi.INT64, 1), (capi.AGG_SUM, capi.INT64, 2),
            (capi.AGG_SUM, capi.INT64, 3), (capi.AGG_AVG, capi.INT64, 0), (capi.AGG_AVG, capi.INT64, 1),
            (capi.AGG_AVG, capi.INT64, 4), (capi.AGG_COUNT_STAR, capi.INT64, -1)]
    batch = ops.Batch.wrap(ctx, [(t.data_ptr(), ty) for t, ty in zip(cols, types)], args.q1_rows, keepalive=cols)
    result["q1"] = profile_workload(torch, ops, ctx, lambda: ops.HashAggregate(ctx, types[:2], desc),
                                    lambda a: a.sink(batch, [0, 1], [2, 3, 4, 5, 6]), args.steps, args.warmup,
                                    args.trace_steps)
    result["q1"]["rows"] = args.q1_rows
    batch.free()
    del q1, cols, batch
    torch.cuda.empty_cache()

    # SSB Q4.1 shape: (i32, u8) keys, 35 groups, one sum
    d = gen.ssb(args.ssb_rows)
    cols, types = [d["year"], d["nation"], d["profit"]], [capi.INT32, capi.UINT8, capi.INT64]
    sdesc = [(capi.AGG_SUM, capi.INT64, 0)]
    batch = ops.Batch.wrap(ctx, [(t.data_ptr(), ty) for t, ty in zip(cols, types)], args.ssb_rows, keepalive=cols)
    result["ssb"] = profile_workload(torch, ops, ctx, lambda: ops.HashAggregate(ctx, types[:2], sdesc),
                                     lambda a: a.sink(batch, [0, 1], [2]), args.steps, args.warmup, args.trace_steps)
    result["ssb"]["rows"] = args.ssb_rows
    batch.free()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
