"""bench.py's synthetic columns are defined as DuckDB SQL and restated with torch ops (bench_data.py): both arms of the
benchmark must see the same rows.  Pinned here against the columns the reference computed from the SQL (stored as
digests in tests/golden/reference_results.json by tests/golden/make_golden.py)."""
import numpy as np
import pytest
import torch

import bench_data as BD
from conftest import assert_column


@pytest.mark.parametrize("offset", [0, 591_855_000 * 3 + 12345])
def test_q1_columns_match_reference(reference_results, offset):
    n = 50_000
    ref = reference_results["bench_data"][f"q1_{offset}"]   # BD.q1_table_sql("t", n, offset)
    got = BD.Gen(torch, "cpu", chunk=7777).q1(n, offset)
    assert set(ref) == set(got)
    for k in ("rf", "ls", "qty", "price", "disc_price", "charge", "disc"):
        assert_column(got[k].numpy(), ref[k], k)
    assert set(np.unique(got["rf"].numpy())) == {65, 78, 82} and set(np.unique(got["ls"].numpy())) == {70, 79}


def test_other_tables_match_reference(reference_results):
    n, nb, groups = 40_000, 1000, 5000
    g = BD.Gen(torch, "cpu", chunk=9999)
    # the reference ran BD.<name>_table_sql with the same arguments
    for name, got in (("ssb", g.ssb(n, 77)), ("q3", g.q3(n, groups, 5)), ("probe", g.probe(n, nb, 3)),
                      ("part", g.part(nb, 1001)), ("scan", g.scan(n, 9))):
        ref = reference_results["bench_data"][name]
        assert set(ref) == set(got), name
        for k, v in ref.items():
            assert_column(got[k].numpy(), v, (name, k))


def test_effective_cores():
    cores, info = BD.effective_cores()
    assert 1 <= cores <= info["sched_affinity"]
