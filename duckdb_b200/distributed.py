"""Multi-GPU plumbing: key-radix shuffle of column batches with torch.distributed (NCCL over NVLink on the GPU
box, gloo in the CPU tests).  One process per GPU.

The ONLY collective on the data path is the partition shuffle (BASELINE.json north_star):
  rank r keeps the rows whose DuckDB radix partition (hash >> (48 - bits)) & (world - 1) == r
  (RadixPartitioning::ApplyMask, src/include/duckdb/common/radix_partitioning.hpp:45-61, with
  bits = log2(world): for 8 GPUs the top 3 of DuckDB's radix bits, SURVEY.md 8e)
so that afterwards every rank builds / probes / aggregates its key range locally with no further exchange -
the multi-GPU analogue of DuckDB's per-partition second phase (radix_partitioned_hashtable.cpp:1229-1305).

exchange_partitions() is backend-agnostic (torch tensors in, torch tensors out) and is what the gloo tests
exercise; shuffle_batch() feeds it from the CUDA radix_partition kernel.
"""
import numpy as np
import torch
import torch.distributed as dist


def log2_world(world):
    bits = int(world).bit_length() - 1
    if (1 << bits) != world:
        raise ValueError("world size must be a power of two for the radix shuffle")
    return bits


def exchange_partitions(columns, counts, group=None):
    """columns: list of 1-D tensors whose rows are grouped by destination rank (partition p = rows
    [sum(counts[:p]), sum(counts[:p+1])) ); counts: per-destination row counts (len == world).
    Returns (received columns, per-source row counts).  Two collectives: the counts all-to-all, then one
    all_to_all_single per column."""
    world = dist.get_world_size(group)
    dev = columns[0].device if columns else torch.device("cpu")
    send = torch.as_tensor(np.asarray(counts, dtype=np.int64), device=dev)
    recv = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_to_all_single(recv, send, group=group)
    send_l = [int(x) for x in send.tolist()]
    recv_l = [int(x) for x in recv.tolist()]
    total = sum(recv_l)
    out = []
    for c in columns:
        o = torch.empty(total, dtype=c.dtype, device=dev)
        dist.all_to_all_single(o, c.contiguous(), output_split_sizes=recv_l, input_split_sizes=send_l, group=group)
        out.append(o)
    if dev.type == "cuda":
        # The send buffers are views of memory owned by the b200 stream-ordered pool (not by torch's allocator): make
        # sure NCCL is done with them before the caller frees / reuses that memory.  (Without this,
        # back-to-back shuffles race with the next partition kernel and silently drop rows.)
        torch.cuda.synchronize(dev)
    return out, recv_l


def allgather_columns(columns, group=None):
    """Replicate a (small) relation on every rank: columns is a list of 1-D tensors with the SAME length on every
    rank; returns the list of concatenated columns (rank 0's rows first).  One all-gather per column.

    This is the other multi-GPU join plan of SURVEY.md 8e: when the build side is small next to the probe side
    (SSB dimensions, TPC-H part / customer) it is cheaper to replicate it and leave the probe side where it is
    than to shuffle both sides by key radix - the reference makes the same choice per thread (every thread probes
    ONE shared hash table, physical_hash_join.cpp:2140-2209)."""
    world = dist.get_world_size(group)
    out = []
    for c in columns:
        c = c.contiguous()
        o = torch.empty(world * c.numel(), dtype=c.dtype, device=c.device)
        dist.all_gather_into_tensor(o, c, group=group)
        out.append(o)
    return out


def choose_join_plan(world, build_bytes_per_rank, probe_bytes_per_rank):
    """'broadcast' when replicating the build side moves fewer bytes per GPU than shuffling both sides:
    (world - 1) x build  vs  (world - 1) / world x (build + probe)."""
    if world <= 1:
        return "local"
    replicate = (world - 1) * build_bytes_per_rank
    shuffle = (world - 1) / world * (build_bytes_per_rank + probe_bytes_per_rank)
    return "broadcast" if replicate <= shuffle else "shuffle"


class _DevArray:
    """zero-copy view of a device buffer for torch.as_tensor (__cuda_array_interface__)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


_TORCH_DTYPE = {1: torch.uint8, 2: torch.uint8, 3: torch.int8, 4: torch.uint16, 5: torch.int16, 6: torch.uint32,
                7: torch.int32, 8: torch.uint64, 9: torch.int64, 11: torch.float32, 12: torch.float64}

_TYPESTR = {1: "|u1", 2: "|u1", 3: "|i1", 4: "<u2", 5: "<i2", 6: "<u4", 7: "<i4", 8: "<u8", 9: "<i8", 11: "<f4",
            12: "<f8"}


def batch_columns_as_tensors(batch, device):
    """torch views (no copy) of the flat, non-NULL columns of a b200 batch."""
    n = batch.nrows
    cols = []
    for i in range(batch.ncols):
        info = batch.column_info(i)
        if info.validity:
            raise ValueError("the radix shuffle handles non-NULL columns only")
        if n == 0:
            cols.append(torch.empty(0, dtype=_TORCH_DTYPE[info.type], device=device))
            continue
        t = torch.as_tensor(_DevArray(info.data, n, _TYPESTR[info.type]), device=device)
        cols.append(t)
    return cols


def shuffle_batch(ctx, batch, key_cols, group=None):
    """Exchange the rows of `batch` so that every rank ends up with the rows of its key-radix partition.
    -> (Batch of the rows this rank owns, keepalive).  Default: the one-kernel peer scatter (PeerShuffle) when every
    column is flat without NULLs and symmetric memory is available; else (or with B200_SHUFFLE=nccl) the CUDA
    radix_partition kernel + NCCL all-to-all.  The result of the peer path lives in the shuffle's receive buffers and
    is valid until the next shuffle of the same column types."""
    from . import capi
    from . import operators as ops

    world = dist.get_world_size(group)
    bits = log2_world(world)
    dev = torch.device("cuda", ctx.device)
    infos = [batch.column_info(i) for i in range(batch.ncols)]
    flat = all(i.vector_type == 0 and not i.validity for i in infos) and bits <= 4
    if flat and dev.type == "cuda":
        ps = peer_shuffle_for(ctx, [i.type for i in infos], batch.nrows, group)
        if ps is not None:
            try:
                out = ps.shuffle(batch, key_cols)
            except capi.B200Error as ex:
                # skew (SURVEY 8 e4, correctness level): a hot key made one partition larger than the receive buffers
                # (sized for 1.25 x the even share).  The rows that did not fit were dropped AND counted, every rank saw
                # the same flag and the same largest partition: grow the buffers to it and shuffle again.
                needed = getattr(ex, "rows_needed", 0)
                if ex.code != capi.ERR_CAPACITY or not needed:
                    raise
                ps = peer_shuffle_for(ctx, [i.type for i in infos], needed, group)
                if ps is None:
                    raise
                out = ps.shuffle(batch, key_cols)
            return out, ps.buffers
    part, counts = ops.radix_partition(ctx, batch, key_cols, bits)
    cols = batch_columns_as_tensors(part, dev)
    types = [part.column_info(i).type for i in range(part.ncols)]
    recv_cols, _ = exchange_partitions(cols, counts, group)
    n = int(recv_cols[0].shape[0]) if recv_cols else 0
    out = ops.Batch.wrap(ctx, [(t.data_ptr(), ty) for t, ty in zip(recv_cols, types)], n, keepalive=recv_cols)
    return out, recv_cols


def allgather_agg_states(ctx, agg, final_agg, max_groups=64, group=None):
    """Low-cardinality multi-GPU aggregate (TPC-H Q1, SSB): every rank packs its partial states into one fixed-size
    device buffer (b200_agg_export_packed: group count + flags, key BIT PATTERNS, NULL-key bits, raw UINT64 state
    columns), ONE NCCL all-gather moves them, and ONE kernel per rank merges all of them into `final_agg`
    (b200_agg_combine_packed) - the multi-GPU form of GroupedAggregateHashTable::Combine
    (aggregate_hashtable.cpp:1168-1197).  Nothing is read back by the host: a rank that holds more than max_groups
    groups flags its buffer and final_agg.finalize() raises B200Error(ERR_CAPACITY), the signal to take the radix
    shuffle instead.  The context's stream must be torch's current stream (as in bench.py) so that the export kernel,
    the collective and the combine kernel are stream-ordered; otherwise the context is synchronised in between."""
    world = dist.get_world_size(group)
    dev = torch.device("cuda", ctx.device)
    words = agg.packed_words(max_groups)
    key = (ctx.device, words, world)
    bufs = _PACKED_BUFFERS.get(key)
    if bufs is None:
        bufs = (torch.empty(words, dtype=torch.int64, device=dev), torch.empty(world * words, dtype=torch.int64, device=dev))
        _PACKED_BUFFERS.clear()
        _PACKED_BUFFERS[key] = bufs
    mine, every = bufs
    same_stream = getattr(ctx, "stream", None) == torch.cuda.current_stream(dev).cuda_stream
    agg.export_packed(mine.data_ptr(), max_groups)
    if not same_stream:
        ctx.sync()
    dist.all_gather_into_tensor(every, mine, group=group)
    if not same_stream:
        torch.cuda.current_stream(dev).synchronize()
    final_agg.combine_packed(every.data_ptr(), world, max_groups)
    return True


_PACKED_BUFFERS = {}


# ------------------------------------------------------------------------------------------------------------------
# The shuffle as ONE kernel per source GPU that scatters partition runs straight into the destination GPUs' receive
# buffers over NVLink peer memory (b200_partition_scatter_dev).  Only the per-partition COUNTS go through a collective;
# there is no intermediate partitioned copy, no NCCL payload all-to-all and no host round trip until the very end.
def peer_write_offsets(count_matrix, rank):
    """count_matrix[s][d] = rows source s sends to destination d.  Rows of lower-ranked sources come first in every
    destination, so source `rank` starts at the column sums over the sources before it.
    -> (offsets[d] for this source, rows this rank receives, rows every rank receives)."""
    m = np.asarray(count_matrix, dtype=np.int64)
    offsets = m[:rank].sum(axis=0).astype(np.uint64)
    totals = m.sum(axis=0)
    return offsets, int(totals[rank]), totals


class PeerShuffle:
    """Receive buffers in symmetric (peer-mapped) memory, one per column, re-used by every shuffle of batches with
    the same column types.  shuffle(), everything stream-ordered on the context's stream (= torch's current stream):
      b200_partition_count_dev -> all-gather of the W x W count matrix -> write offsets (device) -> tiny all-reduce
      ("every rank is done with what the previous shuffle delivered") -> b200_partition_scatter_dev with the peers'
      buffer pointers -> tiny all-reduce ("every source's kernel has completed") -> ONE D2H of (rows received, rows
      dropped) to size the result batch."""

    def __init__(self, ctx, types, capacity_rows, group=None):
        import torch.distributed._symmetric_memory as symm_mem

        self.ctx, self.types, self.capacity = ctx, list(types), int(capacity_rows)
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.bits = log2_world(self.world)
        dev = torch.device("cuda", ctx.device)
        self.dev = dev
        self.buffers, self.handles, self.peer_ptrs = [], [], []
        from . import capi

        for t in self.types:
            buf = symm_mem.empty(self.capacity * capi.TYPE_SIZE[t], dtype=torch.uint8, device=dev)
            hdl = symm_mem.rendezvous(buf, self.group)
            self.buffers.append(buf)
            self.handles.append(hdl)
            self.peer_ptrs.append([int(p) for p in hdl.buffer_ptrs])
        w = self.world
        self.counts = torch.zeros(w, dtype=torch.int64, device=dev)
        self.matrix = torch.zeros(w * w, dtype=torch.int64, device=dev)
        self.offsets = torch.zeros(16, dtype=torch.int64, device=dev)
        self.result = torch.zeros(2, dtype=torch.int64, device=dev)   # [rows received, rows dropped]
        self.flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.dst = [self.peer_ptrs[c][d] for d in range(w) for c in range(len(self.types))]

    def shuffle(self, batch, key_cols):
        from . import capi
        from . import operators as ops

        if getattr(self.ctx, "stream", None) != torch.cuda.current_stream(self.dev).cuda_stream:
            raise capi.B200Error(capi.ERR_INVALID, "PeerShuffle: the context must enqueue on torch's current stream")
        w, r = self.world, self.rank
        ops.partition_count_dev(self.ctx, batch, key_cols, self.bits, self.counts.data_ptr())
        dist.all_gather_into_tensor(self.matrix, self.counts, group=self.group)
        m = self.matrix.view(w, w)
        self.offsets[:w] = m[:r].sum(dim=0) if r else 0
        self.result[0] = m[:, r].sum()
        self.result[1] = 0
        dist.all_reduce(self.flag, group=self.group)    # nobody still reads what the previous shuffle delivered
        ops.partition_scatter_dev(self.ctx, batch, key_cols, self.bits, self.dst, self.offsets.data_ptr(), self.capacity,
                                  self.result[1:].data_ptr())
        dist.all_reduce(self.flag, group=self.group)    # every source's kernel is complete: all rows have landed
        n_recv, dropped = (int(x) for x in self.result.tolist())   # the one host synchronisation
        # a drop anywhere means some receive buffer was too small: every rank must learn about it
        # (a second tiny collective, but on data that is already on the host side of the one synchronisation above)
        bad = torch.tensor([dropped + (1 if n_recv > self.capacity else 0), n_recv], dtype=torch.int64, device=self.dev)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=self.group)
        flag, largest = (int(x) for x in bad.tolist())
        if flag:
            err = capi.B200Error(capi.ERR_CAPACITY, f"PeerShuffle: receive capacity {self.capacity} rows exceeded "
                                                    f"(largest partition: {largest} rows)")
            err.rows_needed = largest    # the same on every rank: shuffle_batch re-sizes the buffers and repeats
            raise err
        return ops.Batch.wrap(self.ctx, [(b.data_ptr(), t) for b, t in zip(self.buffers, self.types)], n_recv,
                              keepalive=self.buffers)


_PEER_SHUFFLES = {}


def peer_shuffle_for(ctx, types, rows_hint, group=None):
    """cached PeerShuffle for (column types, capacity class); None when symmetric memory is unavailable or disabled"""
    import os

    if os.environ.get("B200_SHUFFLE", "peer") != "peer":
        return None
    world = dist.get_world_size(group)
    cap = int(rows_hint * 1.25) + 65536
    key = (ctx.device, tuple(types))
    cur = _PEER_SHUFFLES.get(key)
    # capacities must agree on every rank: take the maximum hint
    t = torch.tensor([cap], dtype=torch.int64, device=torch.device("cuda", ctx.device))
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    cap = int(t.item())
    if cur is not None and cur.capacity >= cap and cur.world == world:
        return cur
    try:
        _PEER_SHUFFLES.pop(key, None)
        cur = PeerShuffle(ctx, types, cap, group)
    except Exception as ex:  # no symmetric memory on this system: the NCCL all-to-all path is used
        import sys

        sys.stderr.write(f"[duckdb_b200] peer shuffle unavailable ({type(ex).__name__}: {ex}); using NCCL all-to-all\n")
        os.environ["B200_SHUFFLE"] = "nccl"
        return None
    _PEER_SHUFFLES[key] = cur
    return cur


# ------------------------------------------------------------------------------------------------------------------
# Shuffle join, pipelined: the probe side is shuffled in chunks on a SECOND stream while the previous chunk is probed on
# the operator's stream - the NVLink transfer (the bound of the shuffle: (N-1)/N of the probe bytes cross NVLink) hides behind the probe kernel instead of adding to it.
class PipelinedShuffleProbe:
    """probe(batch, key_cols, lhs_cols, consume): for every chunk of `batch`: peer-shuffle it (double-buffered receive
    buffers, own context + stream, driven by a helper thread) and probe the rows this rank received with `join`
    (caller's context / thread); consume(out_batch, count) is called per chunk on the caller's thread."""

    def __init__(self, ctx, join, types, rows, nchunks=8, group=None):
        from . import operators as ops

        self.ctx, self.join, self.types, self.group = ctx, join, list(types), group
        self.dev = torch.device("cuda", ctx.device)
        self.nchunks = max(2, int(nchunks))
        self.chunk_rows = (int(rows) + self.nchunks - 1) // self.nchunks
        self.chunk_rows = (self.chunk_rows + 2047) // 2048 * 2048
        self.stream = torch.cuda.Stream(device=self.dev)
        self.sctx = ops.Context(ctx.device, self.stream.cuda_stream)   # the shuffle's own context on its own stream
        cap = int(self.chunk_rows * 1.3) + 65536
        t = torch.tensor([cap], dtype=torch.int64, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        with torch.cuda.stream(self.stream):
            self.shuffles = [PeerShuffle(self.sctx, self.types, int(t.item()), group) for _ in range(2)]
        self.stream.synchronize()

    def probe(self, batch, key_cols, lhs_cols, consume):
        import queue
        import threading

        from . import capi
        from . import operators as ops

        n = batch.nrows
        infos = [batch.column_info(i) for i in range(batch.ncols)]
        chunks = [(lo, min(n, lo + self.chunk_rows)) for lo in range(0, max(n, 1), self.chunk_rows)]
        # every rank must run the same number of exchanges
        t = torch.tensor([len(chunks)], dtype=torch.int64, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        nex = int(t.item())
        ready = queue.Queue()
        free = [threading.Semaphore(1), threading.Semaphore(1)]
        failure = []

        def shuffler():
            try:
                torch.cuda.set_device(self.dev)
                with torch.cuda.stream(self.stream):
                    for c in range(nex):
                        lo, hi = chunks[c] if c < len(chunks) else (n, n)
                        sub = ops.Batch.wrap(self.sctx, [(i.data + lo * capi.TYPE_SIZE[i.type], i.type) for i in infos], hi - lo)
                        free[c & 1].acquire()                      # the probe of chunk c-2 has released this buffer
                        got = self.shuffles[c & 1].shuffle(sub, key_cols)
                        ready.put((c, got))
                ready.put(None)
            except BaseException as ex:  # noqa: BLE001 - handed to the caller's thread
                failure.append(ex)
                ready.put(None)

        th = threading.Thread(target=shuffler, daemon=True)
        th.start()
        total = 0
        error = None
        while True:
            item = ready.get()
            if item is None:
                break
            c, got = item
            try:
                if error is None and got.nrows:
                    out, cnt = self.join.execute(got, key_cols, lhs_cols)   # synchronous on the operator's stream
                    total += cnt
                    consume(out, cnt)
            except BaseException as ex:  # noqa: BLE001 - keep the exchanges going: the peers are inside collectives
                error = ex
            free[c & 1].release()
        th.join()
        if failure:
            raise failure[0]
        if error is not None:
            raise error
        return total
