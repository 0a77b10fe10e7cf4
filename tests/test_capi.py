"""The C-ABI library loads, exports every symbol include/duckdb_b200.h declares, and fails loudly without a GPU."""
import ctypes as C
import os
import re

import pytest

from duckdb_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "duckdb_b200.h")).read()
    return sorted(set(re.findall(r"B200_API\s+[\w\s\*]+?\b(b200_\w+)\s*\(", text)))


def test_header_and_binding_agree():
    assert header_symbols() == sorted(capi.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    for sym in header_symbols():
        assert hasattr(L, sym), f"{sym} is declared in include/duckdb_b200.h but not exported"


def test_version_and_error_strings():
    L = capi.lib()
    assert b"sm_90a" in L.b200_version()
    assert isinstance(L.b200_last_error(), bytes)


def test_no_cpu_fallback_without_device():
    """On a box without a GPU every compute path must fail loudly (B200_ERR_NO_DEVICE), never fall back."""
    L = capi.lib()
    if L.b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    rc = L.b200_ctx_create(0, None, C.byref(h))
    assert rc == capi.ERR_NO_DEVICE
    assert b"no CUDA device" in L.b200_last_error()
    from duckdb_b200 import operators as ops

    with pytest.raises(capi.B200Error) as e:
        ops.Context(0)
    assert e.value.code == capi.ERR_NO_DEVICE


def test_argument_validation_needs_no_device():
    """Every entry point rejects NULL handles / out-pointers with B200_ERR_INVALID before it touches CUDA, and the
    destroy / free / accessor functions accept NULL - the shim relies on both (error paths of B200Check and the
    destructors of its global states).  Runs on the CPU box: none of these calls reaches a kernel."""
    L = capi.lib()
    null = None
    h = C.c_void_p()
    n64 = C.c_uint64()
    assert L.b200_ctx_create(0, null, null) == capi.ERR_INVALID
    assert b"out is NULL" in L.b200_last_error()
    assert L.b200_ctx_sync(null) == capi.ERR_INVALID
    assert L.b200_ctx_stats(null, null, null, null) == capi.ERR_INVALID
    assert L.b200_host_alloc(null, 16, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_batch_upload(null, null, 0, 0, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_batch_wrap(null, null, 0, 0, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_batch_column(null, 0, null) == capi.ERR_INVALID
    assert L.b200_batch_download(null, null, 0, null, null) == capi.ERR_INVALID
    assert L.b200_batch_rows(null) == 0 and L.b200_batch_cols(null) == 0
    assert L.b200_hash(null, null, null, 0, null) == capi.ERR_INVALID
    assert L.b200_filter_project(null, null, null, 0, -1, null, 0, null, null, null, null) == capi.ERR_INVALID
    kt = capi.i32_array([capi.INT64])
    assert L.b200_agg_create(null, kt, 1, null, 0, 0, C.byref(h)) == capi.ERR_INVALID
    assert b"b200_agg_create" in L.b200_last_error()
    assert L.b200_agg_sink(null, null, null, null) == capi.ERR_INVALID
    assert L.b200_agg_group_count(null, C.byref(n64)) == capi.ERR_INVALID
    assert L.b200_agg_export_states(null, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_agg_combine_states(null, null) == capi.ERR_INVALID
    assert L.b200_agg_finalize(null, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_join_create(null, capi.JOIN_INNER, kt, 1, null, 0, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_join_build_sink(null, null, null, null) == capi.ERR_INVALID
    assert L.b200_join_finalize(null) == capi.ERR_INVALID
    assert L.b200_join_build_rows(null, C.byref(n64)) == capi.ERR_INVALID
    assert L.b200_join_probe(null, null, null, null, 0, 0, C.byref(h), null, C.byref(n64)) == capi.ERR_INVALID
    assert L.b200_radix_partition(null, null, null, 0, 0, C.byref(h), C.byref(n64)) == capi.ERR_INVALID
    assert L.b200_partition_count(null, null, null, 0, 0, C.byref(n64)) == capi.ERR_INVALID
    assert L.b200_partition_scatter(null, null, null, 0, 0, null, C.byref(n64)) == capi.ERR_INVALID
    # NULL-tolerant teardown
    L.b200_batch_free(null)
    L.b200_agg_destroy(null)
    L.b200_join_destroy(null)
    L.b200_ctx_destroy(null)
    assert L.b200_host_free(null, null) == capi.OK
