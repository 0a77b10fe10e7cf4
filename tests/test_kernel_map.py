"""Every __global__ kernel of the fast-path, aggregate, generic filter, join and partition sources is claimed by a case of the GPU module that owns the
source (which asserts, through the kernel trace, that it ran) or excluded there with a reason: a new kernel variant
fails this test until a GPU case covers it."""
import ast
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "duckdb_b200", "csrc")
# GPU test module -> the sources whose kernels its KERNEL_CASES / KERNEL_EXCLUDED must account for
MODULES = {
    "test_gpu_kernel_paths.py": ["filter_tile.cu", "agg_hc.cu", "join_tile.cu"],
    "test_gpu_agg_kernel_paths.py": ["agg_tile.cu", "agg_priv.cu", "agg.cu"],
    "test_gpu_filter_interpreter.py": ["filter.cu"],
    "test_gpu_join_kernels.py": ["join.cu", "hash.cu"],
}

_GLOBAL = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^()]*\)\s*)?(\w+)\s*\(")


def kernels_in(path):
    with open(path) as f:
        text = re.sub(r"//[^\n]*", "", f.read())
    return set(_GLOBAL.findall(text))


def gpu_module(name):
    with open(os.path.join(ROOT, "tests", name)) as f:
        source = f.read()
    tree = ast.parse(source)
    consts, funcs = {}, {}
    for node in tree.body:
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name) and \
                node.targets[0].id in ("KERNEL_CASES", "KERNEL_EXCLUDED"):
            consts[node.targets[0].id] = ast.literal_eval(node.value)
        elif isinstance(node, ast.FunctionDef):
            funcs[node.name] = ast.get_source_segment(source, node)
    return consts["KERNEL_CASES"], consts["KERNEL_EXCLUDED"], funcs


def test_parser_finds_the_known_kernels():
    found = set().union(*(kernels_in(os.path.join(CSRC, s)) for srcs in MODULES.values() for s in srcs))
    for k in ["filter_mask_tile_kernel", "compact_tile_kernel", "filter_fused_tile_kernel", "agg_hc_kernel",
              "agg_hc_simple_kernel", "agg_hc_direct_kernel", "join_probe_tile_kernel", "join_probe_lean2_kernel",
              "agg_fast_kernel", "agg_fastreg_kernel", "agg_mid_kernel", "agg_mid2_kernel", "agg_priv_kernel",
              "agg_wpriv_kernel", "agg_sink_kernel", "agg_rehash_kernel", "agg_fix_cnt_kernel", "agg_list_keys_kernel",
              "agg_export_kernel", "agg_combine_kernel", "agg_export_packed_kernel", "agg_packed_header_kernel",
              "agg_combine_packed_kernel", "fill_u64_kernel3", "filter_mask_kernel", "compact_kernel",
              "tile_scan_local_kernel", "tile_scan_chunks_kernel", "tile_scan_add_kernel", "fill_u64_kernel2",
              "join_append_kernel", "join_append_col_kernel", "join_init_slots_kernel", "join_insert_kernel",
              "join_minmax_kernel", "join_dense_build_kernel", "join_inline_kernel", "join_probe_kernel",
              "fill_u64_kernel4", "hash_kernel", "part_hist_kernel", "part_scatter_index_kernel",
              "part_scatter_col_kernel", "fill_u64_kernel", "exclusive_scan_small_kernel", "part_count_kernel",
              "part_move_staged_kernel", "part_move_reg_kernel"]:
        assert k in found, k


def test_every_source_has_one_owner():
    srcs = [s for v in MODULES.values() for s in v]
    assert len(srcs) == len(set(srcs))
    for s in srcs:
        assert os.path.exists(os.path.join(CSRC, s)), s


def test_every_fast_path_kernel_has_a_gpu_case():
    for module, srcs in MODULES.items():
        cases, excluded, _ = gpu_module(module)
        for src in srcs:
            for k in sorted(kernels_in(os.path.join(CSRC, src))):
                assert k in cases or k in excluded, \
                    f"{src}: kernel {k} has no case in KERNEL_CASES of {module} and no exclusion"
                if k in excluded:
                    assert isinstance(excluded[k], str) and excluded[k].strip(), f"{k}: an exclusion needs a reason"


def test_kernel_cases_name_tests_that_check_the_kernel():
    for module, srcs in MODULES.items():
        cases, excluded, funcs = gpu_module(module)
        known = set().union(*(kernels_in(os.path.join(CSRC, s)) for s in srcs))
        for k in excluded:
            assert k in known, f"KERNEL_EXCLUDED of {module} lists {k}, which is not a kernel of its sources"
        for k, tests in cases.items():
            assert k in known, f"KERNEL_CASES of {module} lists {k}, which is not a kernel of its sources"
            assert k not in excluded, k
            assert tests, k
            for t in tests:
                assert t.startswith("test_") and t in funcs, f"{k}: no test function {t}"
                assert k in funcs[t], f"{t} does not name {k}: it cannot be asserting that the kernel ran"
