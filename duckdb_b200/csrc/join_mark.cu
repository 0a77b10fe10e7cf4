// K4 join_probe, in-order MARK variant (b200_join_probe_mark).
//
// A MARK join yields exactly one row per probe row, in probe order, so the result needs no output cursor: probe row i
// writes mark[i] (one byte) and bit i of the validity words at its own position.  A warp handles 32 consecutive rows
// and stores their validity bits with one ballot (half of a 64-bit validity_t word); there are no atomics and no
// count for the host to read back.
//
// Semantics (ScanStructure::ConstructMarkJoinResult, join_hashtable.cpp:1978-2030; the empty build side:
// PhysicalComparisonJoin::ConstructEmptyJoinResult, physical_comparison_join.cpp:116-150):
//   TRUE  the probe key has a match;
//   NULL  the probe key is NULL, or it has no match and the build side holds a NULL key;
//   FALSE otherwise - and always when the build side is empty (no rows at all), even for a NULL probe key.
//
// Two kernels:
//   join_mark_tile_kernel  one exact key column, FLAT and 16-byte aligned: the key tile (and its validity tile) is
//                          bulk-copied HBM -> shared memory by TMA (tile_pipe.cuh); each thread owns 8 rows of a
//                          2048-row tile and issues their 8 table loads back to back (dense table or first
//                          open-addressing slot) before it resolves any of them;
//   join_mark_kernel       everything else b200_join_create accepts (composite keys, constant / dictionary vectors,
//                          unaligned columns): probe_first per row, same output contract.
#include "join.cuh"
#include "tile_pipe.cuh"
#include <cstring>

#define JM_THREADS 256
#define JM_ROWS 8
#define JM_TILE (JM_THREADS * JM_ROWS)
#define JM_STAGES 3

struct MarkTileArgs {
	JoinView J;
	TileCols tc;
	int key_col, key_valid_col; // tile column indices (key_valid_col -1: no validity mask)
	int key_type;
	uint8_t *mark;
	uint32_t *valid32; // the validity words as 32-bit halves: one per warp and row slice
	uint64_t n;
	int stages;
};

// FAST8: 8-byte integer key (a plain 64-bit load, DuckDB's hash is murmur64 of the value); DENSE: direct-addressed table
template <bool FAST8, bool DENSE>
__global__ void __launch_bounds__(JM_THREADS, 2) join_mark_tile_kernel(const __grid_constant__ MarkTileArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[JM_STAGES];
	const int tid = threadIdx.x, lane = tid & 31;
	const JoinView &J = A.J;
	const uint32_t key_off = A.tc.c[A.key_col].smem_off;
	const int key_valid_col = A.key_valid_col;
	const uint32_t valid_off = key_valid_col >= 0 ? A.tc.c[key_valid_col].smem_off : 0;
	const int key_type = A.key_type;
	const bool build_empty = J.build_empty;
	// a probe row without a match is NULL when the build side holds a NULL key (and is not empty)
	const bool miss_valid = build_empty || !J.build_has_null;
	uint8_t *const mark = A.mark;
	uint32_t *const valid32 = A.valid32;
	tp_tile_loop_sync(A.tc, A.stages, smem_raw, bars, 0, A.n, [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		uint64_t key[JM_ROWS];
		bool knull[JM_ROWS], hit[JM_ROWS];
		// 1. keys, and every row's first table load, back to back
		uint32_t ent[JM_ROWS];
		uint64_t sl[JM_ROWS];
		uint4 sv[JM_ROWS];
		bool pend[JM_ROWS];
#pragma unroll
		for (int k = 0; k < JM_ROWS; k++) {
			uint32_t r = k * JM_THREADS + tid;
			knull[k] = false;
			hit[k] = false;
			pend[k] = false;
			ent[k] = 0;
			if (r < rows_in_tile) {
				if (FAST8) {
					key[k] = *(const uint64_t *)(stage + key_off + (size_t)r * 8);
				} else {
					DCol d;
					d.data = stage + key_off;
					d.sel = nullptr;
					d.validity = nullptr;
					d.type = key_type;
					d.vtype = B200_FLAT_VECTOR;
					key[k] = canonical_key_bits(key_type, col_load_raw(d, r));
				}
				if (key_valid_col >= 0) {
					knull[k] = !((stage[valid_off + (r >> 3)] >> (r & 7)) & 1);
				}
				if (!knull[k] && !build_empty) {
					if (DENSE) {
						uint64_t idx = key[k] - J.dense_min;
						if (idx < J.dense_range) {
							ent[k] = __ldg(&J.dense[idx]);
						}
					} else if (key[k] == EMPTY_KEY) {
						hit[k] = J.slots[J.mask + 1].head != ROW_NONE; // side slot
					} else {
						sl[k] = (FAST8 ? murmur64(key[k]) : hash_raw(key_type, key[k])) & J.mask;
						sv[k] = __ldg((const uint4 *)&J.slots[sl[k]]);
						pend[k] = true;
					}
				}
			}
		}
		// 2. resolve: dense entries are final; open addressing walks on past other keys (linear probing)
#pragma unroll
		for (int k = 0; k < JM_ROWS; k++) {
			if (DENSE) {
				hit[k] = ent[k] != 0;
			} else {
				while (pend[k]) {
					uint64_t skey = ((uint64_t)sv[k].y << 32) | sv[k].x;
					if (skey == key[k]) {
						hit[k] = true;
						pend[k] = false;
					} else if (skey == EMPTY_KEY) {
						pend[k] = false;
					} else {
						sl[k] = (sl[k] + 1) & J.mask;
						sv[k] = __ldg((const uint4 *)&J.slots[sl[k]]);
					}
				}
			}
		}
		// 3. write: a byte per row, one ballot of validity bits per warp and row slice
#pragma unroll
		for (int k = 0; k < JM_ROWS; k++) {
			uint32_t r = k * JM_THREADS + tid;
			bool valid = hit[k] || (knull[k] ? build_empty : miss_valid);
			uint32_t bits = __ballot_sync(0xffffffffu, valid);
			if (r < rows_in_tile) {
				__stcs(mark + row0 + r, (uint8_t)hit[k]);
				if (lane == 0) {
					__stcs(valid32 + ((row0 + r) >> 5), bits);
				}
			}
		}
	});
}

// the in-order generic variant: a warp walks 32 consecutive rows at a time
__global__ void __launch_bounds__(256)
    join_mark_kernel(JoinView J, KeyCols keys, uint64_t n, uint8_t *__restrict__ mark, uint32_t *__restrict__ valid32) {
	const int lane = threadIdx.x & 31;
	const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
	const bool miss_valid = J.build_empty || !J.build_has_null;
	for (uint64_t base = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32 * 32; base < n; base += warps * 32) {
		uint64_t row = base + lane;
		bool hit = false, knull = false;
		if (row < n) {
			uint64_t ckeys[MAX_KEYS];
			uint32_t inl;
			hit = probe_first(J, keys, row, &knull, ckeys, &inl) != ROW_NONE;
			mark[row] = hit;
		}
		uint32_t bits = __ballot_sync(0xffffffffu, hit || (knull ? J.build_empty : miss_valid));
		if (lane == 0) {
			valid32[base >> 5] = bits;
		}
	}
}

template <bool FAST8, bool DENSE>
static int launch_mark_tile(b200_ctx *ctx, const MarkTileArgs &A, size_t smem) {
	// the stage size depends on the key width only: at most 3 x (2048 x 8 + 256) bytes
	static int per_sm = 0;
	if (!per_sm) {
		CUDA_TRY(cudaFuncSetAttribute(join_mark_tile_kernel<FAST8, DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
		                              100 * 1024));
		CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, join_mark_tile_kernel<FAST8, DENSE>, JM_THREADS,
		                                                       JM_STAGES * (JM_TILE * 8 + JM_TILE / 8)));
	}
	uint64_t ntiles = (A.n + JM_TILE - 1) / JM_TILE;
	uint64_t max_grid = (uint64_t)ctx->sm_count * (per_sm > 0 ? per_sm : 1);
	unsigned grid = (unsigned)(ntiles < max_grid ? ntiles : max_grid);
	join_mark_tile_kernel<FAST8, DENSE><<<grid, JM_THREADS, smem, ctx->stream>>>(A);
	return B200_OK;
}

// host: enqueue the MARK probe of n >= 1 rows (keys already checked against the join's key types)
int b200_join_probe_mark_launch(b200_ctx *ctx, const JoinView &J, const KeyCols &keys, uint64_t n, uint8_t *mark,
                                uint64_t *validity) {
	const DCol &k0 = keys.c[0];
	bool tile = J.exact && keys.n == 1 && k0.vtype == B200_FLAT_VECTOR && tile_ptr_ok(k0.data) &&
	            (!k0.validity || tile_ptr_ok(k0.validity));
	if (tile) {
		MarkTileArgs A;
		memset(&A, 0, sizeof(A));
		A.J = J;
		A.key_type = k0.type;
		A.mark = mark;
		A.valid32 = (uint32_t *)validity;
		A.n = n;
		A.tc.c[0].ptr = (const unsigned char *)k0.data;
		A.tc.c[0].width = b200_type_size(k0.type);
		A.tc.n = 1;
		A.key_col = 0;
		A.key_valid_col = -1;
		if (k0.validity) {
			A.tc.c[1].ptr = (const unsigned char *)k0.validity;
			A.tc.c[1].width = 0;
			A.tc.n = 2;
			A.key_valid_col = 1;
		}
		tile_cols_finish(&A.tc, JM_TILE);
		A.stages = JM_STAGES;
		size_t smem = (size_t)A.stages * A.tc.stage_bytes;
		bool fast8 = k0.type == B200_INT64 || k0.type == B200_UINT64;
		int rc = fast8 ? (J.dense ? launch_mark_tile<true, true>(ctx, A, smem) : launch_mark_tile<true, false>(ctx, A, smem))
		               : (J.dense ? launch_mark_tile<false, true>(ctx, A, smem) : launch_mark_tile<false, false>(ctx, A, smem));
		B200_TRY(rc);
	} else {
		int grid = grid_for((n + 31) / 32 * 32, 256, 4, ctx->sm_count * 8);
		join_mark_kernel<<<grid, 256, 0, ctx->stream>>>(J, keys, n, mark, (uint32_t *)validity);
	}
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}
