/*
 * duckdb_b200.h - C ABI of the H100-native operator kernels (libduckdb_b200.so).
 *
 * This is the drop-in boundary for DuckDB's three hot operator paths.  DuckDB
 * has no C-level physical-operator plugin API (its C API, src/include/duckdb.h,
 * only covers scalar/aggregate/table functions), so the reference-side binding
 * is a host C++ PhysicalOperator subclass (integration/, INTEGRATION.md) that
 * converts each DataChunk column (UnifiedVectorFormat {sel,data,validity},
 * src/include/duckdb/common/vector/unified_vector_format.hpp:22-35) into a
 * b200_vector view and forwards to the entry points below.  Every entry point
 * cites the reference interface it replaces.
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types.
 *   - every function returns B200_OK (0) or a negative b200_status;
 *     b200_last_error() returns the thread-local message (the C++ shim turns
 *     it into a duckdb::Exception, see SURVEY.md 8b "Error convention").
 *   - all work is enqueued on the context's CUDA stream; functions that
 *     return a row count to the host synchronise that stream.
 *   - there is NO CPU fallback: without a usable CUDA device every compute
 *     entry point fails with B200_ERR_NO_DEVICE.
 */
#ifndef DUCKDB_B200_H
#define DUCKDB_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_API __attribute__((visibility("default")))

typedef enum b200_status {
	B200_OK = 0,
	B200_ERR_INVALID = -1,      /* bad argument / unsupported type            */
	B200_ERR_NO_DEVICE = -2,    /* no CUDA device / driver                    */
	B200_ERR_CUDA = -3,         /* CUDA runtime error (message has details)   */
	B200_ERR_OOM = -4,          /* device or pinned allocation failed         */
	B200_ERR_OVERFLOW = -5,     /* DECIMAL/INT64 arithmetic overflow: the shim
	                               raises duckdb::OutOfRangeException like
	                               function/scalar/operator/arithmetic.cpp:999 */
	B200_ERR_CAPACITY = -6      /* output buffer / table capacity exceeded    */
} b200_status;

/* Physical types: same numeric values as duckdb::PhysicalType
 * (src/include/duckdb/common/types.hpp:76-182). */
typedef enum b200_type {
	B200_BOOL = 1,
	B200_UINT8 = 2,
	B200_INT8 = 3,
	B200_UINT16 = 4,
	B200_INT16 = 5,
	B200_UINT32 = 6,
	B200_INT32 = 7,
	B200_UINT64 = 8,
	B200_INT64 = 9,
	B200_FLOAT = 11,
	B200_DOUBLE = 12,
	B200_INT128 = 204
} b200_type;

/* Vector layouts: same values as duckdb::VectorType
 * (src/include/duckdb/common/enums/vector_type.hpp:15-22). */
typedef enum b200_vector_type {
	B200_FLAT_VECTOR = 0,
	B200_CONSTANT_VECTOR = 2,
	B200_DICTIONARY_VECTOR = 3
} b200_vector_type;

/* A column view = DuckDB's UnifiedVectorFormat.
 *   value(i)   = data[ sel ? sel[i] : i ]         (constant: data[0])
 *   is_valid(i)= validity == NULL || bit (sel? sel[i] : i) of validity is 1
 * validity is DuckDB's ValidityMask: uint64 words, bit=1 means valid
 * (src/include/duckdb/common/types/validity_mask.hpp:50,60).
 * FLAT:       data has n values, sel == NULL.
 * CONSTANT:   data has 1 value, sel == NULL, validity bit 0 tells NULL.
 * DICTIONARY: data has dict_size values, sel has n uint32 indices
 *             (sel_t, src/include/duckdb/common/typedefs.hpp:30), validity is
 *             indexed by dictionary position. */
typedef struct b200_vector {
	int32_t type;        /* b200_type */
	int32_t vector_type; /* b200_vector_type */
	const void *data;
	const uint32_t *sel;
	const uint64_t *validity;
	uint64_t dict_size;  /* dictionary only */
} b200_vector;

typedef struct b200_ctx b200_ctx;     /* one CUDA device + stream + memory pool */
typedef struct b200_batch b200_batch; /* device-resident columns, n rows       */

/* ------------------------------------------------------------------ context */
B200_API const char *b200_last_error(void);
B200_API const char *b200_version(void);
/* number of visible CUDA devices (0 when there is no driver/GPU). */
B200_API int b200_device_count(void);
/* stream: an existing cudaStream_t to enqueue on (e.g. the caller's current
 * stream), or NULL to let the context create its own non-blocking stream. */
B200_API int b200_ctx_create(int device, void *stream, b200_ctx **out);
B200_API void b200_ctx_destroy(b200_ctx *ctx);
B200_API int b200_ctx_sync(b200_ctx *ctx);
/* counters since creation: kernels launched, bytes H2D, bytes D2H. */
B200_API int b200_ctx_stats(b200_ctx *ctx, uint64_t *launches, uint64_t *h2d_bytes, uint64_t *d2h_bytes);
/* pinned host staging memory (cudaHostAlloc) for the shim's DataChunk ring.  Released buffers are kept in a
 * process-wide cache (page-locking costs ~0.3 ms per MB; bound: B200_HOST_CACHE_MB, default 8192) and handed out
 * again by b200_host_alloc; b200_host_trim gives the cache back to the OS. */
B200_API int b200_host_alloc(b200_ctx *ctx, size_t bytes, void **out);
B200_API int b200_host_free(b200_ctx *ctx, void *ptr);
B200_API int b200_host_trim(void);

/* ------------------------------------------------------------------ batches */
/* Stage n rows of host columns to HBM (asynchronous cudaMemcpyAsync on the
 * context stream).  Replaces: the DataChunk handed to
 * PhysicalOperator::Sink/Execute (physical_operator.hpp:105,203).  The host
 * memory must stay valid until the next b200_ctx_sync / counting call. */
B200_API int b200_batch_upload(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows,
                               b200_batch **out);
/* Like b200_batch_upload for FLAT vectors, but into device buffers the caller owns and keeps (dev_data[i]: nrows
 * values; dev_validity[i]: (nrows+63)/64 words, needed only for columns with a validity mask): no device allocation
 * on the row path - the DataChunk ring of the DuckDB-side binding uploads its pinned morsels into a persistent device
 * ring with it.  The copies are asynchronous on the context's stream; host and device buffers must stay untouched
 * until the batch has been consumed (the sink / probe calls return after their kernels have read it). */
B200_API int b200_batch_upload_to(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows,
                                  void *const *dev_data, void *const *dev_validity, b200_batch **out);
/* Wrap columns that already live in HBM (pointers are device pointers); no
 * copy, the caller keeps ownership of the memory. */
B200_API int b200_batch_wrap(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows, b200_batch **out);
B200_API uint64_t b200_batch_rows(const b200_batch *b);
B200_API int b200_batch_cols(const b200_batch *b);
/* device view of column i (pointers are device pointers). */
B200_API int b200_batch_column(const b200_batch *b, int col, b200_vector *out);
/* copy column data (flat values) / validity words of column i back to host.  A result of b200_agg_finalize of at
 * most 1 MiB is served from the pinned host copy finalize took of it: a memcpy, no CUDA call. */
B200_API int b200_batch_download(b200_ctx *ctx, const b200_batch *b, int col, void *dst_data,
                                 uint64_t *dst_validity);
B200_API void b200_batch_free(b200_batch *b);

/* ------------------------------------------------------------------ hashing */
/* out_hashes[i] = DuckDB's hash of the key columns of row i.
 * Replaces VectorOperations::Hash / CombineHash
 * (src/common/vector_operations/vector_hash.cpp:504-552; duckdb::Hash<T>
 * src/include/duckdb/common/types/hash.hpp:38-54).  out_hashes is a device
 * pointer of nrows uint64. */
B200_API int b200_hash(b200_ctx *ctx, const b200_batch *b, const int *key_cols, int nkeys, uint64_t *out_hashes);

/* ----------------------------------------------------- filter / projection */
/* Expression program: nodes in topological order (children before parents).
 * Opcode values are duckdb::ExpressionType values
 * (src/include/duckdb/common/enums/expression_type.hpp) where one exists. */
typedef enum b200_expr_op {
	B200_EXPR_COLREF = 227,   /* BOUND_REF: column `col` of the input batch       */
	B200_EXPR_CONST = 75,     /* VALUE_CONSTANT                                    */
	B200_EXPR_NOT = 13,
	B200_EXPR_IS_NULL = 14,
	B200_EXPR_IS_NOT_NULL = 15,
	B200_EXPR_EQ = 25,
	B200_EXPR_NE = 26,
	B200_EXPR_LT = 27,
	B200_EXPR_GT = 28,
	B200_EXPR_LE = 29,
	B200_EXPR_GE = 30,
	B200_EXPR_DISTINCT = 37,
	B200_EXPR_NOT_DISTINCT = 40,
	B200_EXPR_AND = 50,
	B200_EXPR_OR = 51,
	/* arithmetic (DECIMAL is physical int) and numeric casts: rules below b200_expr_node */
	B200_EXPR_ADD = 1001,
	B200_EXPR_SUB = 1002,
	B200_EXPR_MUL = 1003,
	B200_EXPR_CAST = 1004     /* numeric cast of `left` to `type`                  */
} b200_expr_op;

/* limits of one b200_filter_project call (programs beyond them return B200_ERR_INVALID) */
#define B200_MAX_EXPR_NODES 24
#define B200_MAX_PROJECTIONS 12

typedef struct b200_expr_node {
	int32_t op;       /* b200_expr_op */
	int32_t type;     /* result type (b200_type); comparisons/logic: B200_BOOL */
	int32_t left;     /* child node index or -1 */
	int32_t right;    /* child node index or -1 */
	int32_t col;      /* COLREF: input column */
	int32_t is_null;  /* CONST: 1 = NULL constant */
	union {
		int64_t i;
		uint64_t u;
		double d;
		float f;
	} value;          /* CONST payload; an integer constant must be representable in `type` */
} b200_expr_node;
/* The two operands of a comparison (EQ .. GE, DISTINCT, NOT_DISTINCT) must have the same type;
 * b200_filter_project returns B200_ERR_INVALID otherwise.
 *
 * ADD, SUB, MUL: both operands have the node's type (B200_ERR_INVALID otherwise; BOOL is not allowed).  On
 * integers `col` selects the overflow check, made only for rows whose operands are not NULL and only where the
 * expression is evaluated (projections: surviving rows only); a failed check makes the call return
 * B200_ERR_OVERFLOW:
 *   0  none: the result wraps to the width of its type (AddOperator, add.cpp)
 *   1  the range of the type (TryAddOperator / TrySubtractOperator / TryMultiplyOperator)
 *   2  the DECIMAL bound of the type: 9999 (INT16), 999999999 (INT32), 10^18 - 1 (INT64); other types
 *      return B200_ERR_INVALID (DecimalAddOverflowCheck etc., arithmetic.cpp:975-1008)
 * FLOAT / DOUBLE arithmetic is IEEE in the node's type, rounded once.
 *
 * CAST, like TryCastWithOverflowCheck (numeric_cast.hpp:27-72,187-197):
 *   integer -> integer  the value must lie in the target's range (any signedness, any width), else overflow
 *   integer -> BOOL     value != 0
 *   integer -> FLOAT / DOUBLE  rounded once to nearest even
 *   DOUBLE -> FLOAT     rounded to nearest; a finite value that becomes infinite is an overflow (NaN and
 *                       infinities pass through)
 *   FLOAT / DOUBLE -> integer  not supported: B200_ERR_INVALID */

/* One pass of PhysicalFilter (+ the PhysicalProjection above it):
 *   rows for which node `filter_root` is TRUE (not NULL, not false) survive
 *   (ExpressionExecutor::SelectExpression, expression_executor.cpp:309-325;
 *   NULL -> false: comparison_operators.hpp:199-209);
 *   the output batch holds, for the surviving rows IN INPUT ORDER,
 *   column j = value of node proj_roots[j]  (flat vectors + validity).
 * filter_root = -1 keeps every row (pure projection).
 * out_sel (device, capacity >= nrows uint32, may be NULL): surviving row ids,
 *   the `true_sel` SelectionVector of BinaryExecutor::Select.
 * out_mask (device, (nrows+63)/64 uint64 words, may be NULL): bit i = row i survives.
 * out_count (host): number of surviving rows.
 * Replaces PhysicalFilter::ExecuteInternal (physical_filter.cpp:53-64) and
 * PhysicalProjection::Execute (physical_projection.cpp:34-39). */
B200_API int b200_filter_project(b200_ctx *ctx, const b200_batch *in, const b200_expr_node *nodes, int nnodes,
                                 int filter_root, const int *proj_roots, int nproj, b200_batch **out,
                                 uint32_t *out_sel, uint64_t *out_mask, uint64_t *out_count);

/* ---------------------------------------------------------- hash aggregate */
typedef enum b200_agg_func {
	B200_AGG_COUNT_STAR = 0,
	B200_AGG_COUNT = 1,
	B200_AGG_SUM = 2,             /* integer input -> INT128 (hugeint) sum; double -> double */
	B200_AGG_SUM_NO_OVERFLOW = 3, /* integer input -> INT64 sum (sum_no_overflow)           */
	B200_AGG_MIN = 4,
	B200_AGG_MAX = 5,
	B200_AGG_AVG = 6              /* -> DOUBLE; integer input: long double(hugeint)/count    */
} b200_agg_func;

typedef struct b200_agg_desc {
	int32_t func;       /* b200_agg_func */
	int32_t input_type; /* b200_type of the argument (ignored for COUNT_STAR) */
	int32_t input;      /* which aggregate-input column this aggregate reads: index into the input_cols[]
	                       list given to b200_agg_sink (like the BOUND_REF of a DuckDB aggregate into the
	                       aggregate_input_chunk, physical_hash_aggregate.cpp:433-451).  Aggregates with the
	                       same `input` share state (sum(x) and avg(x) keep ONE 128-bit sum).  -1 for COUNT_STAR */
	int32_t reserved;
} b200_agg_desc;

typedef struct b200_agg b200_agg; /* = GlobalSinkState of PhysicalHashAggregate */

/* Replaces PhysicalHashAggregate's sink state / GroupedAggregateHashTable
 * construction (physical_hash_aggregate.cpp:128-189; aggregate_hashtable.cpp).
 * expected_groups is a hint (0 = unknown); the table grows as needed. */
B200_API int b200_agg_create(b200_ctx *ctx, const int32_t *key_types, int nkeys, const b200_agg_desc *aggs,
                             int naggs, uint64_t expected_groups, b200_agg **out);
/* Like b200_agg_create; filters[a] = -1 (no filter) or the index, in the input_cols list of b200_agg_sink, of a
 * B200_BOOL column: aggregate a sees only the rows where that column is valid and nonzero (FILTER (WHERE ...),
 * physical_hash_aggregate.cpp:361-404).  filters == NULL is b200_agg_create.
 * Every row still creates its group: SUM / MIN / MAX / AVG over no passing rows are NULL, COUNT is 0, and
 * COUNT_STAR with filter f counts the rows where f is valid and nonzero.
 * Aggregates share state exactly when they have the same (input, filter) pair: sum(x) and sum(x) FILTER (p) keep
 * two sums.  Each distinct pair is one internal input; at most 12 pairs (columns used only as filters do not count).
 * The input_cols list has 1 + max(input, filter) entries and every index must be an input or a filter; a column
 * read both as an input and as a filter must be B200_BOOL.  b200_agg_sink returns B200_ERR_INVALID for a filter
 * column that is not B200_BOOL.  Each sink call folds every filtered pair into one validity mask with one kernel,
 * on the context's stream, in a scratch block it frees stream-ordered after the sink's kernels.
 * b200_agg_export_states / b200_agg_export_packed of an aggregate with filters produce one state block per internal
 * input, in order of first appearance of its pair in `aggs`; without filters (filters NULL or all -1) the blocks
 * follow the input indices, as for b200_agg_create.  b200_agg_combine_states / b200_agg_combine_packed need both
 * aggregates created with identical descs and filters.
 * B200_ERR_INVALID for bad arguments, B200_ERR_NO_DEVICE without a CUDA device (after the arguments are checked). */
B200_API int b200_agg_create_filtered(b200_ctx *ctx, const int32_t *key_types, int nkeys, const b200_agg_desc *aggs,
                                      const int32_t *filters, int naggs, uint64_t expected_groups, b200_agg **out);
/* Sink one batch: find-or-create each row's group and update the aggregate
 * states.  key_cols[k] indexes the key columns of `in`; input_cols[i] is the
 * column of `in` holding aggregate input i (i = b200_agg_desc.input; the list
 * has 1 + max(input) entries, may be NULL when every aggregate is COUNT_STAR).
 * NULL keys form a group (GROUP BY semantics,
 * aggregate_hashtable.cpp:85-88); NULL aggregate inputs are skipped.
 * Replaces PhysicalHashAggregate::Sink (physical_hash_aggregate.cpp:415-470) ->
 * GroupedAggregateHashTable::AddChunk / FindOrCreateGroupsInternal /
 * UpdateAggregates (aggregate_hashtable.cpp:630-642,803-977,688-722). */
B200_API int b200_agg_sink(b200_agg *agg, const b200_batch *in, const int *key_cols, const int *input_cols);
/* Number of groups so far (synchronises). */
B200_API int b200_agg_group_count(b200_agg *agg, uint64_t *out_groups);
/* Export partial state: batch columns = [keys..., per aggregate raw state
 * columns: rows, then per input cnt / sum lo,hi / min / max] (see DESIGN.md
 * "aggregate state columns"), all UINT64, one row per group.  Used
 * for the multi-GPU combine; mirrors the partitioned uncombined rows handed to
 * GroupedAggregateHashTable::Combine (aggregate_hashtable.cpp:1168-1197). */
B200_API int b200_agg_export_states(b200_agg *agg, b200_batch **out);
/* Merge partial states produced by b200_agg_export_states (possibly on another
 * GPU and shuffled here) into this table.
 * Replaces RowOperations::CombineStates (row_aggregate.cpp:120-150). */
B200_API int b200_agg_combine_states(b200_agg *agg, const b200_batch *states);
/* Packed partial states for the low-cardinality multi-GPU combine (TPC-H Q1, SSB): a fixed-size device buffer of
 * b200_agg_packed_words(agg, max_groups) uint64 words per rank - [groups, flags, key bit patterns, NULL-key bits,
 * raw state columns] - so that ONE all-gather (ncclAllGather / all_gather_into_tensor) moves every rank's partial
 * aggregate and ONE kernel merges them.  Both calls are stream-asynchronous and never synchronise with the host;
 * a rank that held more than max_groups groups sets a flag in its buffer and the b200_agg_finalize of the combining
 * aggregate returns B200_ERR_CAPACITY (the caller then takes the b200_agg_export_states / radix-shuffle route).
 * Replaces GroupedAggregateHashTable::Combine (aggregate_hashtable.cpp:1168-1197) across GPUs. */
B200_API uint64_t b200_agg_packed_words(b200_agg *agg, uint64_t max_groups);
B200_API int b200_agg_export_packed(b200_agg *agg, uint64_t *dst_dev, uint64_t max_groups);
B200_API int b200_agg_combine_packed(b200_agg *agg, const uint64_t *src_dev, int nranks, uint64_t max_groups);
/* Finalize: output batch columns = [group keys in key order..., one result
 * column per aggregate], one row per group, row order unspecified
 * (physical_hash_aggregate.hpp:110-112).  Result types: COUNT* -> INT64;
 * SUM(int) -> INT128; SUM_NO_OVERFLOW -> INT64; SUM(float/double) -> DOUBLE;
 * MIN/MAX -> input type; AVG -> DOUBLE.
 * The result is read-only: its columns share one device block, and a result of
 * at most 1 MiB also has a host copy taken at finalize, from which
 * b200_batch_download serves it (writes through b200_batch_column pointers
 * would not reach that copy).
 * Replaces RadixPartitionedHashTable::GetData / RowOperations::FinalizeStates
 * (radix_partitioned_hashtable.cpp:1307-1360,1374-1442). */
B200_API int b200_agg_finalize(b200_agg *agg, b200_batch **out);
B200_API void b200_agg_destroy(b200_agg *agg);

/* ---------------------------------------------------------------- hash join */
typedef enum b200_join_type { /* duckdb::JoinType values (enums/join_type.hpp:18-34) */
	B200_JOIN_LEFT = 1,
	B200_JOIN_RIGHT = 2,
	B200_JOIN_INNER = 3,
	B200_JOIN_OUTER = 4, /* FULL OUTER */
	B200_JOIN_SEMI = 5,
	B200_JOIN_ANTI = 6,
	B200_JOIN_MARK = 7
} b200_join_type;

typedef struct b200_join b200_join; /* = HashJoinGlobalSinkState + JoinHashTable */

/* Replaces PhysicalHashJoin's sink state / JoinHashTable construction
 * (physical_hash_join.cpp:764-834; join_hashtable.cpp).  Conditions are
 * equality on nkeys key columns (NULL keys never match: join_hashtable.cpp:714-742).
 * Key and payload columns: any b200_type except B200_INT128 (B200_ERR_INVALID);
 * 1..8 key columns, 0..12 payload columns. */
B200_API int b200_join_create(b200_ctx *ctx, int join_type, const int32_t *key_types, int nkeys,
                              const int32_t *payload_types, int npayload, b200_join **out);
/* Append build-side rows.  Replaces PhysicalHashJoin::Sink -> JoinHashTable::Build
 * (join_hashtable.cpp:617-712). */
B200_API int b200_join_build_sink(b200_join *join, const b200_batch *in, const int *key_cols,
                                  const int *payload_cols);
/* Build the hash table over everything sunk so far.  Replaces
 * PhysicalHashJoin::Finalize -> JoinHashTable::Finalize / InsertHashesLoop
 * (physical_hash_join.cpp:1893-2022; join_hashtable.cpp:1113-1139,858-984). */
B200_API int b200_join_finalize(b200_join *join);
B200_API int b200_join_build_rows(b200_join *join, uint64_t *out_rows);
/* Probe one batch.  Output batch columns =
 *   [ lhs_cols of the probe batch gathered for each result row ...,
 *     build payload columns gathered for each result row ... ]
 * (join_hashtable.cpp:1757-1759 column order).  out_lhs_sel (device, may be
 * NULL, capacity = out_capacity) receives the probe row id of each result row.
 * INNER: one result row per (probe row, matching build row).
 * LEFT:  like INNER plus unmatched probe rows with NULL payload.
 * SEMI / ANTI: probe rows with (without) a match, lhs columns only.
 * MARK: every probe row, one extra BOOL column (NULL when the probe key is
 *       NULL) after the lhs columns.
 * RIGHT: like INNER; OUTER (FULL): like LEFT.  Both also flag every build row
 *       they emit, for b200_join_scan_unmatched.  A call that returns
 *       B200_ERR_CAPACITY may have flagged rows already; its retry emits the
 *       same rows, so the flags end up the same.
 * out_capacity bounds the result rows (B200_ERR_CAPACITY if exceeded; pass 0
 * to let the library size it exactly with a counting pass).
 * Probe key columns have the types the join was created with; lhs columns
 * (at most 12) may be of any b200_type except B200_INT128 (B200_ERR_INVALID),
 * and flat, constant or dictionary vectors, like the keys.
 * Result order is unspecified (SURVEY.md 3.3).
 * Replaces PhysicalHashJoin::ExecuteInternal -> JoinHashTable::Probe /
 * ScanStructure::Next* / GatherRHS (physical_hash_join.cpp:2140-2209;
 * join_hashtable.cpp:1178-1209,1476-1837,1690-1730). */
B200_API int b200_join_probe(b200_join *join, const b200_batch *probe, const int *key_cols, const int *lhs_cols,
                             int nlhs, uint64_t out_capacity, b200_batch **out, uint32_t *out_lhs_sel,
                             uint64_t *out_count);
/* Probe one batch of a finalized B200_JOIN_MARK join IN PROBE ORDER: for probe
 * row i, mark_dev[i] (device, nrows bytes, BOOL 0 / 1) and bit i of
 * mark_validity_dev (device, (nrows+63)/64 uint64 words, DuckDB validity_t
 * words, bit = 1 valid; bits past row nrows-1 are unspecified):
 *   TRUE  the probe key has a match;
 *   NULL  the probe key is NULL, or it has no match and the build side holds a
 *         NULL key;
 *   FALSE otherwise, and for every row (NULL keys too) when the build side is
 *         empty.
 * Same key columns as b200_join_probe; no lhs columns are copied.  The call is
 * stream-asynchronous: it enqueues one kernel on the context's stream and
 * returns without synchronising.  B200_ERR_INVALID for a NULL argument, a join
 * of another type or one not yet finalized; B200_ERR_NO_DEVICE without a CUDA
 * device.  Replaces JoinHashTable::ConstructMarkJoinResult
 * (join_hashtable.cpp:1978-2030) behind PhysicalHashJoin::ExecuteInternal
 * (physical_hash_join.cpp:2140-2209) for MARK joins, and
 * PhysicalComparisonJoin::ConstructEmptyJoinResult
 * (physical_comparison_join.cpp:116-150) for an empty build side. */
B200_API int b200_join_probe_mark(b200_join *join, const b200_batch *probe, const int *key_cols, uint8_t *mark_dev,
                                  uint64_t *mark_validity_dev);
/* B200_JOIN_RIGHT / B200_JOIN_OUTER, after the probes: the build rows in [row_begin, row_end) that no
 * b200_join_probe call matched (NULL-key rows included), in build-row order.  Output batch = the build
 * payload columns; out_build_rows (device, may be NULL) receives each result row's build row index;
 * out_count (host).  Synchronises.  row_begin must be a multiple of 64.
 * The caller emits these rows with NULL probe-side columns.  B200_ERR_INVALID for a NULL argument, a join of
 * another type, one not yet finalized, or a range that is not inside [0, b200_join_build_rows) or whose
 * row_begin is not a multiple of 64; B200_ERR_NO_DEVICE without a CUDA device.  Replaces
 * JoinHashTable::ScanFullOuter (join_hashtable.cpp:2302-2356) behind PhysicalHashJoin::GetData
 * (physical_hash_join.cpp) for RIGHT and FULL OUTER joins. */
B200_API int b200_join_scan_unmatched(b200_join *join, uint64_t row_begin, uint64_t row_end,
                                      b200_batch **out, uint32_t *out_build_rows, uint64_t *out_count);
B200_API void b200_join_destroy(b200_join *join);

/* ---------------------------------------------------------- radix partition */
/* Reorder the rows of `in` so that partition p = (hash >> (48 - bits)) & (2^bits - 1)
 * of the key hash is contiguous: RadixPartitioning::ApplyMask
 * (src/include/duckdb/common/radix_partitioning.hpp:45-61).  With bits = 3 the
 * partition id is the GPU rank of an 8-GPU box.  out has the same columns as
 * `in` (flat), rows grouped by partition; counts_host[p] = rows of partition p
 * (2^bits entries).  Row order inside a partition is unspecified.
 * bits 0..12; 1..8 key columns; columns of any b200_type except B200_INT128
 * (B200_ERR_INVALID), flat, constant or dictionary, with or without NULLs.
 * Replaces PartitionedTupleData::AppendUnified (partitioned_tuple_data.cpp:62-96). */
B200_API int b200_radix_partition(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                                  b200_batch **out, uint64_t *counts_host);

/* ------------------------------------------- shuffle without an intermediate copy */
/* EXPERIMENTAL (not yet measured on hardware).  The multi-GPU exchange of
 * PartitionedTupleData::Partition + the cross-thread Combine
 * (partitioned_tuple_data.cpp:62-96,270-290) as two calls around one all-to-all
 * of COUNTS only; the rows themselves are written by the scatter kernel straight
 * into their destination GPU's buffers (NVLink peer memory), no NCCL payload
 * collective and no intermediate partitioned copy.
 *   1. b200_partition_count: counts_host[p] = rows of `in` whose radix partition
 *      (same id as b200_radix_partition) is p.
 *   2. the caller exchanges the counts and derives, per destination p, the row
 *      offset at which THIS source's rows start in p's receive buffers.
 *   3. b200_partition_scatter: every column c of every row of partition p is
 *      stored to dst_cols[p * ncols + c] at row dst_row_offsets[p] + (rank of the
 *      row among this source's rows of partition p; order unspecified).  The
 *      destination pointers may be local or peer-mapped device memory.
 * Restrictions: bits <= 4, 1..16 flat columns without NULLs of at most 48 bytes
 * per row, no B200_INT128 column (the shuffle path; B200_ERR_INVALID otherwise).
 * The _dev forms below have the same restrictions. */
B200_API int b200_partition_count(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                                  uint64_t *counts_host);
B200_API int b200_partition_scatter(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                                    void *const *dst_cols, const uint64_t *dst_row_offsets);

/* Stream-asynchronous forms of the two calls above (no host round trip): the per-partition counts are left in device
 * memory (2^bits words), the write offsets are read from device memory, rows that would land beyond capacity_rows of a
 * destination buffer are NOT written and counted in *dropped_dev (the caller checks it once the exchange is over).
 * The b200_shuffle of SURVEY.md 8b = count_dev -> all-gather of the counts -> scatter_dev, all on one stream. */
B200_API int b200_partition_count_dev(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                                      uint64_t *counts_dev);
B200_API int b200_partition_scatter_dev(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                                        void *const *dst_cols, const uint64_t *dst_row_offsets_dev,
                                        uint64_t capacity_rows, uint64_t *dropped_dev);

#ifdef __cplusplus
}
#endif
#endif /* DUCKDB_B200_H */
