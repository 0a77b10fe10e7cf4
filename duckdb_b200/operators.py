"""Host-side mirror of DuckDB's operator interface for the three hot paths, over the C ABI.

Names and call order follow the reference's PhysicalOperator contract
(src/include/duckdb/execution/physical_operator.hpp:102-254):

  PhysicalFilter / PhysicalProjection : Execute(chunk)                 -> FilterProject.execute
  PhysicalHashAggregate               : Sink* -> Combine -> Finalize -> GetData  -> HashAggregate
  PhysicalHashJoin                    : Sink* (build) -> Finalize -> Execute* (probe) -> HashJoin

A "chunk" here is a list of Vector (flat / constant / dictionary, like
UnifiedVectorFormat) with any number of rows (the shim batches DuckDB's
2048-row DataChunks into morsels before calling the C ABI).  All compute runs
in libduckdb_b200.so on the GPU; nothing here computes results on the host.
"""
import ctypes as C

import numpy as np

from . import capi
from .capi import B200Error, check, lib


class Vector:
    """Host column view = UnifiedVectorFormat {sel, data, validity}."""

    def __init__(self, data, valid=None, vector_type=capi.FLAT_VECTOR, sel=None):
        self.data = np.ascontiguousarray(data)
        if self.data.dtype not in capi.TYPE_OF_DTYPE:
            raise B200Error(capi.ERR_INVALID, f"unsupported dtype {self.data.dtype}")
        self.type = capi.TYPE_OF_DTYPE[self.data.dtype]
        self.valid = None if valid is None else np.ascontiguousarray(valid, dtype=bool)
        self.vector_type = vector_type
        self.sel = None if sel is None else np.ascontiguousarray(sel, dtype=np.uint32)
        self._words = None if self.valid is None else capi.validity_words(self.valid)

    @staticmethod
    def flat(data, valid=None):
        return Vector(data, valid)

    @staticmethod
    def constant(value, dtype, is_null=False):
        return Vector(np.array([value], dtype=dtype), np.array([not is_null]) if is_null else None,
                      capi.CONSTANT_VECTOR)

    @staticmethod
    def dictionary(dictionary, sel, valid=None):
        """valid is indexed by dictionary position (like DuckDB's child validity)."""
        return Vector(dictionary, valid, capi.DICTIONARY_VECTOR, sel)

    def as_struct(self):
        v = capi.Vector()
        v.type = self.type
        v.vector_type = self.vector_type
        v.data = self.data.ctypes.data
        v.sel = self.sel.ctypes.data if self.sel is not None else None
        v.validity = self._words.ctypes.data if self._words is not None else None
        v.dict_size = len(self.data) if self.vector_type == capi.DICTIONARY_VECTOR else 0
        return v

    def logical(self, n):
        """Materialise (values, valid) of n rows on the host - used by tests only."""
        if self.vector_type == capi.FLAT_VECTOR:
            idx = np.arange(n)
        elif self.vector_type == capi.CONSTANT_VECTOR:
            idx = np.zeros(n, dtype=np.int64)
        else:
            idx = self.sel[:n].astype(np.int64)
        vals = self.data[idx]
        valid = np.ones(n, dtype=bool) if self.valid is None else self.valid[idx]
        return vals, valid


class Context:
    """One GPU + stream (b200_ctx)."""

    def __init__(self, device=0, stream=None):
        """stream: None -> the context creates a private non-blocking stream; a CUDA stream handle -> the context
        enqueues on it.  Handle 0 (what torch.cuda.current_stream().cuda_stream returns for torch's default stream)
        is passed on as cudaStreamLegacy (0x1): a NULL handle would mean "create your own" to b200_ctx_create, and
        the kernels would silently run UNORDERED with torch's / NCCL's work (rows get lost in a multi-GPU shuffle)."""
        self.handle = C.c_void_p()
        handle = None if stream is None else C.c_void_p(int(stream) if int(stream) != 0 else 1)
        check(lib().b200_ctx_create(device, handle, C.byref(self.handle)))
        self.device = device
        self.stream = None if stream is None else int(stream)   # as torch reports it (0 = the default stream)

    def sync(self):
        check(lib().b200_ctx_sync(self.handle))

    def stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().b200_ctx_stats(self.handle, C.byref(a), C.byref(b), C.byref(c)))
        return {"launches": a.value, "h2d_bytes": b.value, "d2h_bytes": c.value}

    def close(self):
        if self.handle:
            lib().b200_ctx_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Batch:
    """Device-resident columns (b200_batch)."""

    def __init__(self, ctx, handle, keepalive=None):
        self.ctx = ctx
        self.handle = handle
        self._keepalive = keepalive

    @staticmethod
    def upload(ctx, vectors, nrows):
        arr = (capi.Vector * max(1, len(vectors)))(*[v.as_struct() for v in vectors])
        h = C.c_void_p()
        check(lib().b200_batch_upload(ctx.handle, arr, len(vectors), nrows, C.byref(h)))
        return Batch(ctx, h, keepalive=vectors)

    @staticmethod
    def wrap(ctx, columns, nrows, keepalive=None):
        """columns already in HBM: (device_ptr, b200_type[, validity_device_ptr]) for a flat column, or
        (dictionary_ptr, b200_type, validity_ptr_or_None, sel_device_ptr, dict_size) for a dictionary vector
        (validity is indexed by dictionary position, like DuckDB's)."""
        arr = (capi.Vector * max(1, len(columns)))()
        for i, col in enumerate(columns):
            arr[i].type = col[1]
            arr[i].data = col[0]
            arr[i].validity = col[2] if len(col) > 2 and col[2] else None
            if len(col) > 3:
                arr[i].vector_type = capi.DICTIONARY_VECTOR
                arr[i].sel = col[3]
                arr[i].dict_size = col[4]
            else:
                arr[i].vector_type = capi.FLAT_VECTOR
                arr[i].sel = None
                arr[i].dict_size = 0
        h = C.c_void_p()
        check(lib().b200_batch_wrap(ctx.handle, arr, len(columns), nrows, C.byref(h)))
        return Batch(ctx, h, keepalive=keepalive)

    @property
    def nrows(self):
        return lib().b200_batch_rows(self.handle)

    @property
    def ncols(self):
        return lib().b200_batch_cols(self.handle)

    def column_info(self, col):
        v = capi.Vector()
        check(lib().b200_batch_column(self.handle, col, C.byref(v)))
        return v

    def download(self, col):
        """-> (values ndarray, valid bool ndarray).  INT128 columns come back as python ints (object array)."""
        info = self.column_info(col)
        n = self.nrows
        if info.type == capi.INT128:
            raw = np.zeros(2 * n, dtype=np.uint64)
        else:
            raw = np.zeros(n, dtype=capi.DTYPE_OF_TYPE[info.type])
        words = np.zeros((n + 63) // 64, dtype=np.uint64)
        check(lib().b200_batch_download(self.ctx.handle, self.handle, col, raw.ctypes.data if n else None,
                                        words.ctypes.data if n else None))
        valid = capi.valid_from_words(words, n) if n else np.zeros(0, dtype=bool)
        if info.type == capi.INT128:
            lo = raw[0::2]
            hi = raw[1::2].view(np.int64)
            vals = np.array([int(l) + (int(h) << 64) for l, h in zip(lo, hi)], dtype=object)
            return vals, valid
        return raw, valid

    def download_into(self, col, data_ptr, validity_ptr=None):
        """D2H of column `col` into caller-owned host memory (use pinned memory for full PCIe speed)."""
        check(lib().b200_batch_download(self.ctx.handle, self.handle, col, C.c_void_p(data_ptr),
                                        C.c_void_p(validity_ptr) if validity_ptr else None))

    def download_all(self):
        return [self.download(i) for i in range(self.ncols)]

    def free(self):
        if self.handle:
            lib().b200_batch_free(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def hash_keys(ctx, batch, key_cols, out_dev_ptr):
    """VectorOperations::Hash/CombineHash of the key columns into a device uint64 buffer."""
    check(lib().b200_hash(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), C.c_void_p(out_dev_ptr)))


# ---------------------------------------------------------------- expressions
class Expr:
    """Tiny builder for b200_expr_node programs (children before parents)."""

    def __init__(self):
        self.nodes = []

    def _add(self, op, type_, left=-1, right=-1, col=0, is_null=0, value=None):
        n = capi.ExprNode()
        n.op, n.type, n.left, n.right, n.col, n.is_null = op, type_, left, right, col, is_null
        if value is not None:
            if type_ == capi.DOUBLE:
                n.value.d = float(value)
            elif type_ == capi.FLOAT:
                n.value.u = int(np.array([value], dtype=np.float32).view(np.uint32)[0])
            elif type_ in (capi.UINT64, capi.UINT32, capi.UINT16, capi.UINT8, capi.BOOL):
                n.value.u = int(value)
            else:
                n.value.i = int(value)
        self.nodes.append(n)
        return len(self.nodes) - 1

    def col(self, index, type_):
        return self._add(capi.EXPR_COLREF, type_, col=index)

    def const(self, value, type_, is_null=False):
        return self._add(capi.EXPR_CONST, type_, is_null=1 if is_null else 0, value=0 if is_null else value)

    def cmp(self, op, left, right):
        return self._add(op, capi.BOOL, left, right)

    def and_(self, left, right):
        return self._add(capi.EXPR_AND, capi.BOOL, left, right)

    def or_(self, left, right):
        return self._add(capi.EXPR_OR, capi.BOOL, left, right)

    def not_(self, child):
        return self._add(capi.EXPR_NOT, capi.BOOL, child)

    def is_null(self, child):
        return self._add(capi.EXPR_IS_NULL, capi.BOOL, child)

    def is_not_null(self, child):
        return self._add(capi.EXPR_IS_NOT_NULL, capi.BOOL, child)

    def arith(self, op, type_, left, right, check_mode=1):
        """check_mode: 0 none, 1 integer range of type_, 2 DECIMAL bound of type_."""
        return self._add(op, type_, left, right, col=check_mode)

    def cast(self, child, type_):
        return self._add(capi.EXPR_CAST, type_, child)

    def array(self):
        return (capi.ExprNode * max(1, len(self.nodes)))(*self.nodes)


class FilterProject:
    """PhysicalFilter (+ PhysicalProjection): Execute(input) -> surviving rows of the projected expressions.

    Mirrors PhysicalFilter::ExecuteInternal (physical_filter.cpp:53-64) and
    PhysicalProjection::Execute (physical_projection.cpp:34-39)."""

    def __init__(self, ctx, expr, filter_root, proj_roots):
        self.ctx, self.expr, self.filter_root, self.proj_roots = ctx, expr, filter_root, list(proj_roots)

    def execute(self, batch, want_sel=False, want_mask=False, sel_dev=None, mask_dev=None):
        """-> (out Batch or None, count, sel ndarray|None, mask words ndarray|None).
        sel_dev / mask_dev: optional caller-owned device buffers (pointers)."""
        import torch  # device scratch for the optional sel / mask outputs (plumbing only)

        n = batch.nrows
        sel_t = mask_t = None
        if want_sel and sel_dev is None:
            sel_t = torch.empty(max(n, 1), dtype=torch.int32, device=f"cuda:{self.ctx.device}")
            sel_dev = sel_t.data_ptr()
        if want_mask and mask_dev is None:
            mask_t = torch.empty(max((n + 63) // 64, 1), dtype=torch.int64, device=f"cuda:{self.ctx.device}")
            mask_dev = mask_t.data_ptr()
        out = C.c_void_p()
        count = C.c_uint64()
        nodes = self.expr.array()
        check(lib().b200_filter_project(self.ctx.handle, batch.handle, nodes, len(self.expr.nodes), self.filter_root,
                                        capi.int_array(self.proj_roots), len(self.proj_roots), C.byref(out),
                                        C.c_void_p(sel_dev) if sel_dev else None,
                                        C.c_void_p(mask_dev) if mask_dev else None, C.byref(count)))
        ob = Batch(self.ctx, out) if out else None
        sel = mask = None
        if sel_t is not None:
            sel = sel_t[:count.value].cpu().numpy().view(np.uint32)
        if mask_t is not None:
            mask = mask_t[:(n + 63) // 64].cpu().numpy().view(np.uint64)
        return ob, count.value, sel, mask


class HashAggregate:
    """PhysicalHashAggregate: Sink -> (Combine) -> Finalize/GetData.

    Mirrors PhysicalHashAggregate::{Sink,Combine,Finalize,GetDataInternal}
    (physical_hash_aggregate.cpp:415,503,838,958)."""

    def __init__(self, ctx, key_types, aggs, expected_groups=0):
        """aggs: list of (func, input_type, input) - `input` is the index of the aggregate's argument in the
        input_cols list passed to sink() (aggregates over the same column share it); -1 for COUNT_STAR.
        2-tuples (func, input_type) get one input each, in order."""
        self.ctx = ctx
        self.key_types = list(key_types)
        full, nxt = [], 0
        for a in aggs:
            if len(a) == 3:
                full.append(tuple(a))
            elif a[0] == capi.AGG_COUNT_STAR:
                full.append((a[0], a[1], -1))
            else:
                full.append((a[0], a[1], nxt))
                nxt += 1
        self.aggs = full
        self.ninputs = 1 + max([a[2] for a in full] + [-1])
        descs = (capi.AggDesc * max(1, len(full)))()
        for i, (f, t, inp) in enumerate(full):
            descs[i].func, descs[i].input_type, descs[i].input, descs[i].reserved = f, t, inp, 0
        self.handle = C.c_void_p()
        check(lib().b200_agg_create(ctx.handle, capi.i32_array(self.key_types), len(self.key_types), descs, len(aggs),
                                    expected_groups, C.byref(self.handle)))

    def sink(self, batch, key_cols, input_cols):
        """input_cols[i] = batch column of aggregate input i."""
        assert len(input_cols) == self.ninputs, (len(input_cols), self.ninputs)
        check(lib().b200_agg_sink(self.handle, batch.handle, capi.int_array(key_cols), capi.int_array(input_cols)))

    def group_count(self):
        g = C.c_uint64()
        check(lib().b200_agg_group_count(self.handle, C.byref(g)))
        return g.value

    def export_states(self):
        out = C.c_void_p()
        check(lib().b200_agg_export_states(self.handle, C.byref(out)))
        return Batch(self.ctx, out)

    def combine_states(self, states_batch):
        check(lib().b200_agg_combine_states(self.handle, states_batch.handle))

    def packed_words(self, max_groups):
        return int(lib().b200_agg_packed_words(self.handle, max_groups))

    def export_packed(self, dst_dev_ptr, max_groups):
        """partial states -> one fixed-size device buffer (stream-asynchronous, no host round trip)"""
        check(lib().b200_agg_export_packed(self.handle, C.c_void_p(dst_dev_ptr), max_groups))

    def combine_packed(self, src_dev_ptr, nranks, max_groups):
        """merge nranks packed buffers (consecutive in device memory, e.g. the output of one all-gather)"""
        check(lib().b200_agg_combine_packed(self.handle, C.c_void_p(src_dev_ptr), nranks, max_groups))

    def finalize(self):
        out = C.c_void_p()
        check(lib().b200_agg_finalize(self.handle, C.byref(out)))
        return Batch(self.ctx, out)

    def close(self):
        if self.handle:
            lib().b200_agg_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HashJoin:
    """PhysicalHashJoin: Sink (build side) -> Finalize -> Execute (probe side).

    Mirrors PhysicalHashJoin::{Sink,Finalize,ExecuteInternal} (physical_hash_join.cpp:764,1893,2140)."""

    def __init__(self, ctx, join_type, key_types, payload_types):
        self.ctx = ctx
        self.join_type = join_type
        self.key_types, self.payload_types = list(key_types), list(payload_types)
        self.handle = C.c_void_p()
        check(lib().b200_join_create(ctx.handle, join_type, capi.i32_array(self.key_types), len(self.key_types),
                                     capi.i32_array(self.payload_types), len(self.payload_types),
                                     C.byref(self.handle)))

    def sink(self, batch, key_cols, payload_cols):
        check(lib().b200_join_build_sink(self.handle, batch.handle, capi.int_array(key_cols),
                                         capi.int_array(payload_cols)))

    def finalize(self):
        check(lib().b200_join_finalize(self.handle))

    def build_rows(self):
        r = C.c_uint64()
        check(lib().b200_join_build_rows(self.handle, C.byref(r)))
        return r.value

    def execute(self, batch, key_cols, lhs_cols, out_capacity=0, lhs_sel_dev=None):
        out = C.c_void_p()
        count = C.c_uint64()
        check(lib().b200_join_probe(self.handle, batch.handle, capi.int_array(key_cols), capi.int_array(lhs_cols),
                                    len(lhs_cols), out_capacity, C.byref(out),
                                    C.c_void_p(lhs_sel_dev) if lhs_sel_dev else None, C.byref(count)))
        return Batch(self.ctx, out), count.value

    def close(self):
        if self.handle:
            lib().b200_join_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def radix_partition(ctx, batch, key_cols, bits):
    """-> (Batch with rows grouped by partition, counts ndarray[2^bits]).

    Partition id = (hash >> (48 - bits)) & (2^bits - 1): RadixPartitioning::ApplyMask
    (radix_partitioning.hpp:45-61)."""
    out = C.c_void_p()
    counts = np.zeros(1 << bits, dtype=np.uint64)
    check(lib().b200_radix_partition(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), bits,
                                     C.byref(out), counts.ctypes.data_as(C.POINTER(C.c_uint64))))
    return Batch(ctx, out), counts


def partition_count(ctx, batch, key_cols, bits):
    """Pass 1 of the copy-free shuffle (EXPERIMENTAL, b200_partition_count): rows per radix partition."""
    counts = np.zeros(1 << bits, dtype=np.uint64)
    check(lib().b200_partition_count(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), bits,
                                     counts.ctypes.data_as(C.POINTER(C.c_uint64))))
    return counts


def partition_scatter(ctx, batch, key_cols, bits, dst_ptrs, dst_row_offsets):
    """Pass 2 (EXPERIMENTAL, b200_partition_scatter): dst_ptrs[p * ncols + c] = device pointer (local or peer-mapped)
    of column c in partition p's destination, dst_row_offsets[p] = first row this source may write there."""
    nparts, ncols = 1 << bits, batch.ncols
    if len(dst_ptrs) != nparts * ncols or len(dst_row_offsets) != nparts:
        raise B200Error(capi.ERR_INVALID, "partition_scatter: need 2^bits x ncols pointers and 2^bits offsets")
    ptrs = (C.c_void_p * len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_ptrs])
    offs = np.ascontiguousarray(dst_row_offsets, dtype=np.uint64)
    check(lib().b200_partition_scatter(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), bits,
                                       ptrs, offs.ctypes.data_as(C.POINTER(C.c_uint64))))


def partition_count_dev(ctx, batch, key_cols, bits, counts_dev_ptr):
    """rows per radix partition into device memory (2^bits uint64 words), stream-asynchronous"""
    check(lib().b200_partition_count_dev(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), bits,
                                         C.c_void_p(counts_dev_ptr)))


def partition_scatter_dev(ctx, batch, key_cols, bits, dst_ptrs, offsets_dev_ptr, capacity_rows, dropped_dev_ptr):
    """the fused partition + transfer kernel with its write offsets in device memory, stream-asynchronous"""
    nparts, ncols = 1 << bits, batch.ncols
    if len(dst_ptrs) != nparts * ncols:
        raise B200Error(capi.ERR_INVALID, "partition_scatter_dev: need 2^bits x ncols pointers")
    ptrs = (C.c_void_p * len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_ptrs])
    check(lib().b200_partition_scatter_dev(ctx.handle, batch.handle, capi.int_array(key_cols), len(key_cols), bits, ptrs,
                                           C.c_void_p(offsets_dev_ptr), capacity_rows, C.c_void_p(dropped_dev_ptr)))
