"""b200_agg_create_filtered's argument checks, which need no device, and the kernel map of agg_filter.cu: every __global__
kernel there is claimed by a case of tests/test_gpu_agg_filter.py that asserts, through the kernel trace, that it ran."""
import ctypes as C
import os

import pytest

from duckdb_b200 import capi
from test_kernel_map import CSRC, gpu_module, kernels_in

MAX_INPUTS = 12


def _descs(aggs):
    arr = (capi.AggDesc * max(1, len(aggs)))()
    for i, (f, t, inp) in enumerate(aggs):
        arr[i].func, arr[i].input_type, arr[i].input, arr[i].reserved = f, t, inp, 0
    return arr


def _create(aggs, filters, ctx=True, keys=(capi.INT64,)):
    """-> (status, last error) of b200_agg_create_filtered with a dummy context pointer: every case here fails in the
    host-side checks, before the context is read"""
    L = capi.lib()
    dummy = (C.c_uint64 * 64)()
    h = C.c_void_p()
    rc = L.b200_agg_create_filtered(C.cast(dummy, C.c_void_p) if ctx else None, capi.i32_array(list(keys)), len(keys),
                                    _descs(aggs), capi.i32_array(filters) if filters is not None else None, len(aggs),
                                    0, C.byref(h))
    return rc, L.b200_last_error()


def test_null_arguments_are_invalid():
    L = capi.lib()
    h = C.c_void_p()
    kt = capi.i32_array([capi.INT64])
    descs = _descs([(capi.AGG_SUM, capi.INT64, 0)])
    flt = capi.i32_array([1])
    dummy = (C.c_uint64 * 64)()
    ctx = C.cast(dummy, C.c_void_p)
    assert L.b200_agg_create_filtered(None, kt, 1, descs, flt, 1, 0, C.byref(h)) == capi.ERR_INVALID
    assert b"b200_agg_create_filtered: bad arguments" in L.b200_last_error()
    assert L.b200_agg_create_filtered(ctx, kt, 1, descs, flt, 1, 0, None) == capi.ERR_INVALID
    assert L.b200_agg_create_filtered(ctx, None, 1, descs, flt, 1, 0, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_agg_create_filtered(ctx, kt, 1, None, flt, 1, 0, C.byref(h)) == capi.ERR_INVALID
    assert L.b200_agg_create_filtered(ctx, kt, 0, descs, flt, 1, 0, C.byref(h)) == capi.ERR_INVALID


@pytest.mark.parametrize("bad", [-2, 2 * MAX_INPUTS, 1 << 30])
def test_filter_index_out_of_range(bad):
    rc, err = _create([(capi.AGG_SUM, capi.INT64, 0)], [bad])
    assert rc == capi.ERR_INVALID
    assert b"filter column" in err and b"out of range" in err


def test_input_index_out_of_range():
    rc, err = _create([(capi.AGG_SUM, capi.INT64, 2 * MAX_INPUTS)], [0])
    assert rc == capi.ERR_INVALID and b"out of range" in err


def test_input_cols_must_be_dense():
    """column 1 is neither an input nor a filter: the list 0..2 has a hole"""
    rc, err = _create([(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_COUNT, capi.INT64, 0)], [2, -1])
    assert rc == capi.ERR_INVALID and b"dense" in err
    rc, err = _create([(capi.AGG_COUNT_STAR, capi.INT64, -1)], [1])
    assert rc == capi.ERR_INVALID and b"column 0" in err


def _no_device():
    return capi.lib().b200_device_count() <= 0


def test_more_than_max_inputs_pairs():
    """one input under 13 different filters is 13 internal inputs"""
    aggs = [(capi.AGG_SUM, capi.INT64, 0)] * (MAX_INPUTS + 1)
    rc, err = _create(aggs, list(range(1, MAX_INPUTS + 2)))
    assert rc == capi.ERR_INVALID and b"pairs" in err


@pytest.mark.skipif(not _no_device(), reason="passes the host checks: with a device it would read the dummy context")
def test_max_inputs_pairs_pass_the_host_checks():
    """12 pairs of one input, and 12 inputs each under its own filter (24 columns, 12 pairs: filter columns do not
    count towards the limit), get as far as the device check"""
    aggs = [(capi.AGG_SUM, capi.INT64, 0)] * MAX_INPUTS
    rc, err = _create(aggs, list(range(1, MAX_INPUTS + 1)))
    assert rc == capi.ERR_NO_DEVICE, err
    aggs = [(capi.AGG_SUM, capi.INT64, i) for i in range(MAX_INPUTS)]
    rc, err = _create(aggs, [MAX_INPUTS + i for i in range(MAX_INPUTS)])
    assert rc == capi.ERR_NO_DEVICE, err


def test_a_filter_column_read_as_another_type_is_invalid():
    """column 1 is a filter of one aggregate and a BIGINT input of another, in both orders"""
    for aggs, filters in [([(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_SUM, capi.INT64, 1)], [1, -1]),
                          ([(capi.AGG_SUM, capi.INT64, 1), (capi.AGG_SUM, capi.INT64, 0)], [-1, 1])]:
        rc, err = _create(aggs, filters)
        assert rc == capi.ERR_INVALID and b"column 1" in err and b"type" in err, err


def test_layout_checks_still_apply():
    rc, err = _create([(capi.AGG_SUM_NO_OVERFLOW, capi.DOUBLE, 0)], [1])
    assert rc == capi.ERR_INVALID and b"sum_no_overflow" in err
    rc, err = _create([(99, capi.INT64, 0)], [1])
    assert rc == capi.ERR_INVALID and b"unknown aggregate function" in err


def test_no_device():
    """with valid arguments and no CUDA device the call fails with B200_ERR_NO_DEVICE (no CPU fallback), before it
    reads the context - which could not have been created without a device"""
    if not _no_device():
        pytest.skip("a CUDA device is present: tests/test_gpu_agg_filter.py creates filtered aggregates")
    for filters in ([1, -1], [-1, -1], None):
        rc, err = _create([(capi.AGG_SUM, capi.INT64, 0), (capi.AGG_COUNT_STAR, capi.INT64, -1)], filters)
        assert rc == capi.ERR_NO_DEVICE, filters
        assert b"no CUDA device" in err


def test_every_filter_kernel_has_a_gpu_case():
    cases, excluded, funcs = gpu_module("test_gpu_agg_filter.py")
    kernels = kernels_in(os.path.join(CSRC, "agg_filter.cu"))
    assert kernels == {"agg_filter_fold_kernel"}
    for k in kernels:
        assert k in cases or (k in excluded and excluded[k].strip()), k
    for k, tests in cases.items():
        assert k in kernels and tests, k
        for t in tests:
            assert t in funcs and k in funcs[t], f"{t} does not name {k}: it cannot be asserting that the kernel ran"
