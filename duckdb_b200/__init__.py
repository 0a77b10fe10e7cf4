"""duckdb_b200: H100-native kernels for DuckDB's hash-join, hash-aggregate and filter/projection operators.

The product is duckdb_b200/_lib/libduckdb_b200.so (CUDA sm_90a + C ABI, include/duckdb_b200.h);
this package is the thin host-side mirror of the reference's operator interface over that ABI.
"""
from . import capi  # noqa: F401
from .capi import B200Error  # noqa: F401

__version__ = "0.1"
