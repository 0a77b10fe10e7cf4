"""b200_join_scan_unmatched's argument checks, which need no device, the two new join types against DuckDB's JoinType
values, and the kernel map of join_outer.cu: every __global__ kernel there is claimed by a case of
tests/test_gpu_join_outer.py that asserts, through the kernel trace, that it ran."""
import ctypes as C
import os
import subprocess

import pytest

from duckdb_b200 import capi
from test_kernel_map import CSRC, gpu_module, kernels_in

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_null_arguments_are_invalid():
    """the join handle, out and out_count may not be NULL (out_build_rows may): B200_ERR_INVALID before anything else
    is looked at"""
    L = capi.lib()
    dummy = (C.c_uint64 * 64)()
    p = C.cast(dummy, C.c_void_p)
    out, count = C.c_void_p(), C.c_uint64()
    args = [p, 0, 64, C.byref(out), None, C.byref(count)]
    for i in (0, 3, 5):
        a = list(args)
        a[i] = None
        assert L.b200_join_scan_unmatched(*a) == capi.ERR_INVALID, i
        assert b"b200_join_scan_unmatched: bad arguments" in L.b200_last_error()


def test_no_device():
    """with every argument present and no CUDA device the call fails with B200_ERR_NO_DEVICE (no CPU fallback), before
    it reads the join handle - which could not have been created without a device"""
    L = capi.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_gpu_join_outer.py checks the join type, finalize and range rules")
    dummy = (C.c_uint64 * 64)()
    p = C.cast(dummy, C.c_void_p)
    out, count = C.c_void_p(), C.c_uint64()
    for rows in (None, p):
        assert L.b200_join_scan_unmatched(p, 0, 64, C.byref(out), rows, C.byref(count)) == capi.ERR_NO_DEVICE
        assert b"no CUDA device" in L.b200_last_error()


def test_join_types_are_duckdbs(tmp_path, reference_results):
    """B200_JOIN_RIGHT and B200_JOIN_OUTER, as a C99 compiler sees the header and as capi declares them, are DuckDB's
    JoinType::RIGHT and JoinType::OUTER"""
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text('#include <stdio.h>\n#include "duckdb_b200.h"\n'
                   'int main(void) { printf("%d %d\\n", (int)B200_JOIN_RIGHT, (int)B200_JOIN_OUTER); return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           str(src), "-o", str(exe)])
    right, outer = map(int, subprocess.check_output([str(exe)], text=True).split())
    join = reference_results["enums"]["JoinType"]
    assert (right, outer) == (join["RIGHT"], join["OUTER"]) == (capi.JOIN_RIGHT, capi.JOIN_OUTER) == (2, 4)


def test_scan_is_exported():
    assert "b200_join_scan_unmatched" in capi.EXPORTED_SYMBOLS
    assert capi.lib().b200_join_scan_unmatched is not None


def test_every_outer_kernel_has_a_gpu_case():
    cases, excluded, funcs = gpu_module("test_gpu_join_outer.py")
    kernels = kernels_in(os.path.join(CSRC, "join_outer.cu"))
    assert kernels == {"join_rows_offset_kernel"}
    for k in kernels:
        assert k in cases or (k in excluded and excluded[k].strip()), k
    for k, tests in cases.items():
        assert k in kernels and tests, k
        for t in tests:
            assert t in funcs and k in funcs[t], f"{t} does not name {k}: it cannot be asserting that the kernel ran"
