import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100)")


def golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def py_scalar(x):
    """numpy / Python scalar -> the plain Python value the reference's fetchall() returns"""
    if x is None:
        return None
    if isinstance(x, (bool, np.bool_)):
        return bool(x)
    if isinstance(x, (int, np.integer)):
        return int(x)
    return float(x)


def digest(rows):
    """SHA-256 of a canonical list of rows (or values): equal digests <=> equal results, without storing them."""
    canon = [tuple(py_scalar(x) for x in r) if isinstance(r, (tuple, list)) else py_scalar(r) for r in rows]
    return hashlib.sha256(repr(canon).encode()).hexdigest()


def digest_array(a):
    """SHA-256 of an integer column as little-endian 64-bit words"""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a).astype("<i8")).tobytes()).hexdigest()


def bincount_mean(keys, values):
    """per-key mean of `values` in ascending key order (keys that occur only): sum by np.bincount / count"""
    keys = np.asarray(keys)
    s, c = np.bincount(keys, weights=values), np.bincount(keys)
    return s[c > 0] / c[c > 0]


def assert_matches(got, ref, what=""):
    """`got` (a sorted row list) against a stored summary {n, head, tail, sha}: the cheap parts first, so that a
    mismatch says where it is"""
    got = [tuple(py_scalar(x) for x in r) if isinstance(r, (tuple, list)) else (py_scalar(r),) for r in got]
    assert len(got) == ref["n"], (what, "row count", len(got), ref["n"])
    assert [list(r) for r in got[:3]] == ref["head"], (what, "first rows", got[:3], ref["head"])
    assert [list(r) for r in got[-3:]] == ref["tail"], (what, "last rows", got[-3:], ref["tail"])
    assert digest([r if len(r) > 1 else r[0] for r in got]) == ref["sha"], (what, "rows differ (same count, head, tail)")


def assert_column(values, ref, what=""):
    v = np.asarray(values).astype(np.int64)
    assert len(v) == ref["n"] and v[:4].tolist() == ref["head"], (what, v[:4].tolist(), ref["head"])
    assert digest_array(v) == ref["sha"], (what, "values differ (same length and head)")


@pytest.fixture(scope="session")
def reference_results():
    """The reference's answers on the tests' seeded inputs (tests/golden/make_golden.py reference_results)."""
    with open(os.path.join(GOLDEN, "reference_results.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def ctx():
    """One b200 context on cuda:0, enqueueing on torch's current stream (so torch events see our kernels)."""
    import torch
    from duckdb_b200 import operators as ops

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    torch.cuda.set_device(0)
    c = ops.Context(0, torch.cuda.current_stream().cuda_stream)
    yield c
    c.close()
