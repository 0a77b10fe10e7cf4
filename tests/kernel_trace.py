"""Which CUDA kernels ran: a context manager over torch.profiler's CUDA activity trace (CUPTI).

CUPTI records every kernel of the process, including those libduckdb_b200.so launches through ctypes, so a test can
check that the dispatcher picked the kernel variant it meant to exercise rather than a generic fall-back.  The names
are the demangled kernel names without their parameter list, e.g. ``join_probe_lean2_kernel<1, 8, false>``."""
import contextlib
import json
import os
import re
import tempfile
import time

# The profiler keeps only the GPU activities whose timestamps fall inside the window it measures on the host clock, and
# the two clocks disagree by a few milliseconds (a kernel's reported start lay between 2.9 ms before and 3.5 ms after
# its host-side launch on an H100).  A window shorter than that offset, such as one around a single small kernel, can
# lose every kernel.  Idle margins on both sides of the block keep what it launches inside the window.
WINDOW_MARGIN_S = 0.02


def _strip(name):
    """'void f<1, 2>(Args)' -> 'f<1, 2>'"""
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


@contextlib.contextmanager
def kernel_trace():
    """with kernel_trace() as names: ...  -> afterwards `names` holds the kernels launched inside the block, in order"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    names = []
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(WINDOW_MARGIN_S)
        yield names
        torch.cuda.synchronize()
        time.sleep(WINDOW_MARGIN_S)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    names.extend(_strip(e["name"]) for e in sorted((e for e in events if e.get("cat") == "kernel"),
                                                   key=lambda e: e.get("ts", 0)))


def _norm(s):
    return re.sub(r"\s+", "", s)


def ran(names, kernel):
    """did `kernel` run?  A name with template arguments ('f<1, true>') must match them exactly; a bare name
    ('f') matches every instantiation."""
    want = _norm(kernel)
    for n in names:
        n = _norm(n)
        if n == want or ("<" not in want and n.split("<", 1)[0] == want):
            return True
    return False


def assert_ran(names, *kernels):
    for k in kernels:
        assert ran(names, k), f"expected kernel {k} to run; the trace holds {sorted(set(names))}"


def assert_not_ran(names, *kernels):
    for k in kernels:
        assert not ran(names, k), f"kernel {k} ran but should not have; the trace holds {sorted(set(names))}"


def traced(fn):
    """-> (fn(), kernel names).  A window in which the profiler delivered no kernel at all is not evidence about the
    dispatcher: fn, which must be repeatable, runs once more in a fresh window, and a second empty window is an
    error."""
    for attempt in range(2):
        with kernel_trace() as names:
            result = fn()
        if names:
            return result, names
    raise AssertionError("torch.profiler recorded no CUDA kernel in two windows that launched kernels")
