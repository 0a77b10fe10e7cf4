"""b200_join_probe_mark's argument checks, which need no device, and the kernel map of join_mark.cu: every __global__
kernel there is claimed by a case of tests/test_gpu_join_mark.py that asserts, through the kernel trace, that it ran."""
import ctypes as C
import os

import pytest

from duckdb_b200 import capi
from test_kernel_map import CSRC, gpu_module, kernels_in


def test_null_arguments_are_invalid():
    """every NULL argument is rejected with B200_ERR_INVALID before anything else is looked at"""
    L = capi.lib()
    dummy = (C.c_uint64 * 64)()
    p = C.cast(dummy, C.c_void_p)
    keys = capi.int_array([0])
    args = [p, p, keys, p, p]
    for i in range(len(args)):
        a = list(args)
        a[i] = None
        assert L.b200_join_probe_mark(*a) == capi.ERR_INVALID, i
        assert b"b200_join_probe_mark: bad arguments" in L.b200_last_error()


def test_no_device():
    """with every argument present and no CUDA device the call fails with B200_ERR_NO_DEVICE (no CPU fallback), before
    it reads the join handle - which could not have been created without a device"""
    L = capi.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_gpu_join_mark.py checks the join type and finalize rules")
    dummy = (C.c_uint64 * 64)()
    p = C.cast(dummy, C.c_void_p)
    assert L.b200_join_probe_mark(p, p, capi.int_array([0]), p, p) == capi.ERR_NO_DEVICE
    assert b"no CUDA device" in L.b200_last_error()


def test_every_mark_kernel_has_a_gpu_case():
    cases, excluded, funcs = gpu_module("test_gpu_join_mark.py")
    kernels = kernels_in(os.path.join(CSRC, "join_mark.cu"))
    assert kernels == {"join_mark_tile_kernel", "join_mark_kernel"}
    for k in kernels:
        assert k in cases or (k in excluded and excluded[k].strip()), k
    for k, tests in cases.items():
        assert k in kernels and tests, k
        for t in tests:
            assert t in funcs and k in funcs[t], f"{t} does not name {k}: it cannot be asserting that the kernel ran"
