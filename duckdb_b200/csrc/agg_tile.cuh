// Shared front end of the TMA-staged aggregate sink kernels (agg_tile.cu: FAST / FASTREG / MID / MID2,
// agg_priv.cu: PRIV): staged-row access, the global-path fallback of a row and the warp-specialised tile loop.
#pragma once
#include "agg.cuh"
#include "tile_pipe.cuh"

#define AT_THREADS 256
#define AT_TILE 1024
#define AT_MAX_STAGES 3
#define FAST_MAX_SLOTS 16
#define AT_SMEM_BUDGET (222 * 1024)

struct StageMap {
	int key_data[MAX_KEYS], key_valid[MAX_KEYS];
	int in_data[MAX_INPUTS], in_valid[MAX_INPUTS];
};

struct TileArgs {
	AggTable T;
	AggLayout L;
	KeyCols keys;
	AggCols ac;
	TileCols tc;
	StageMap sm;
	int stages;
	uint64_t row_begin, row_end;
	uint32_t *deferred;
	unsigned long long *counters;
};

// ------------------------------------------------------------------ staged row access
__device__ __forceinline__ uint64_t stage_value(const unsigned char *stage, const TileCol &c, int type, uint32_t r) {
	DCol d;
	d.data = stage + c.smem_off;
	d.sel = nullptr;
	d.validity = nullptr;
	d.type = type;
	d.vtype = B200_FLAT_VECTOR;
	return col_load_raw(d, r);
}

__device__ __forceinline__ bool stage_valid(const unsigned char *stage, const TileCols &tc, int vcol, uint32_t r) {
	if (vcol < 0) {
		return true;
	}
	return (stage[tc.c[vcol].smem_off + (r >> 3)] >> (r & 7)) & 1;
}

__device__ __forceinline__ void stage_pack_key(const TileArgs &A, const unsigned char *stage, uint32_t r,
                                               uint64_t kw[KEY_WORDS_MAX]) {
#pragma unroll
	for (int w = 0; w < KEY_WORDS_MAX; w++) {
		kw[w] = 0;
	}
	uint32_t nullbits = 0;
#pragma unroll 1
	for (int j = 0; j < A.L.nkeys; j++) {
		if (stage_valid(stage, A.tc, A.sm.key_valid[j], r)) {
			uint64_t raw = stage_value(stage, A.tc.c[A.sm.key_data[j]], A.L.key_type[j], r);
			pack_field(kw, A.L.key_off[j], key_field_bits(A.L.key_type[j], raw));
		} else {
			nullbits |= 1u << j;
		}
	}
	pack_field(kw, A.L.null_off, (uint64_t)nullbits);
}

// a row that does not fit the per-CTA structure: global path
__device__ __forceinline__ void row_to_global(const TileArgs &A, const unsigned char *stage, uint32_t r, uint64_t row,
                                              const uint64_t kw[KEY_WORDS_MAX]) {
	uint64_t gs = agg_find_or_create(A.T, A.L, hash_packed_key(A.L, kw), kw);
	if (gs == SLOT_DEFER) {
		unsigned long long d = atomicAdd(&A.counters[0], 1ULL);
		A.deferred[d] = (uint32_t)row;
		return;
	}
	uint64_t *grow = A.T.slots + gs * (uint64_t)A.L.stride;
	atomicAdd((unsigned long long *)(grow + A.L.rows_off), 1ULL);
	for (int i = 0; i < A.L.ninputs; i++) {
		if (stage_valid(stage, A.tc, A.sm.in_valid[i], r)) {
			agg_apply_input(A.L, i, grow, stage_value(stage, A.tc.c[A.sm.in_data[i]], A.L.input_type[i], r),
			                A.ac.track_cnt[i]);
		}
	}
}

// The tile loop shared by the aggregate kernels.  BODY(stage, r, row) is called for every row of the CTA's tiles.
// Warp-specialised producer/consumer ring: the CTA is launched with NC consumer threads + ONE extra producer warp.
// The producer's lane 0 walks the CTA's tiles, waits for empty[s] (all consumer warps are done with the stage) and
// issues the TMA bulk copies that complete on full[s]; consumers only ever wait for data, never for each other.
// bars: 2*AT_MAX_STAGES mbarriers (full[], empty[]).
template <class BODY>
__device__ __forceinline__ void tile_loop(const TileArgs &A, unsigned char *stages, uint64_t *bars, int NC, BODY body) {
	const uint32_t TILE = A.tc.tile_rows;
	const uint64_t total = A.row_end - A.row_begin;
	const uint64_t ntiles = (total + TILE - 1) / TILE;
	const uint64_t nfull = total / TILE;
	const int S = A.stages;
	uint64_t *full = bars, *empty = bars + AT_MAX_STAGES;
	if (threadIdx.x == 0) {
		for (int s = 0; s < S; s++) {
			tp_mbar_init(&full[s], 1);
			tp_mbar_init(&empty[s], NC / 32); // one arrival per consumer warp
		}
		tp_fence_mbar_init();
	}
	__syncthreads();
	if ((int)threadIdx.x >= NC) {
		// ---- producer warp
		if ((threadIdx.x & 31) == 0) {
			for (uint64_t k = 0;; k++) {
				uint64_t t = blockIdx.x + k * gridDim.x;
				if (t >= nfull) {
					break;
				}
				int s = (int)(k % S);
				uint64_t use = k / S;
				if (use >= 1) {
					tp_wait(&empty[s], (uint32_t)((use - 1) & 1));
				}
				tp_issue_full(A.tc, stages + (size_t)s * A.tc.stage_bytes, &full[s], A.row_begin + t * TILE);
			}
		}
	} else {
		// ---- consumers
		for (uint64_t k = 0;; k++) {
			uint64_t t = blockIdx.x + k * gridDim.x;
			if (t >= ntiles) {
				break;
			}
			int s = (int)(k % S);
			unsigned char *stage = stages + (size_t)s * A.tc.stage_bytes;
			uint32_t rows_in_tile = TILE;
			uint64_t row0 = A.row_begin + t * TILE;
			if (t < nfull) {
				tp_wait(&full[s], (uint32_t)((k / S) & 1));
			} else {
				// ragged last tile: plain cooperative copy by the consumers (named barrier 1 = consumers only)
				asm volatile("bar.sync 1, %0;" ::"r"(NC) : "memory");
				rows_in_tile = (uint32_t)(total - t * TILE);
				for (int i = 0; i < A.tc.n; i++) {
					const TileCol &c = A.tc.c[i];
					uint32_t bytes = c.width ? rows_in_tile * c.width : (rows_in_tile + 7) / 8;
					const unsigned char *src = c.width ? c.ptr + row0 * c.width : c.ptr + row0 / 8;
					unsigned char *dst = stage + c.smem_off;
					for (uint32_t q = threadIdx.x; q < bytes; q += NC) {
						dst[q] = src[q];
					}
				}
				asm volatile("bar.sync 1, %0;" ::"r"(NC) : "memory");
			}
			for (uint32_t r = threadIdx.x; r < rows_in_tile; r += NC) {
				body(stage, r, row0 + r);
			}
			__syncwarp();
			if ((threadIdx.x & 31) == 0) {
				tp_arrive(&empty[s]);
			}
		}
	}
	__syncthreads();
}

#define REG_MAX_SUMS 6
#define REG_MAX_SLOTS 8

struct RegLayout {
	int nsum;
	int in_of_sum[REG_MAX_SUMS];         // distinct-input index of sum accumulator j
	uint32_t sum_smem_off[REG_MAX_SUMS]; // byte offset of the input's tile inside a stage
	uint32_t sum_unsigned;               // bit j: the input of sum accumulator j is an unsigned integer
	int nkeys;
	uint32_t key_smem_off[MAX_KEYS];
	uint32_t key_width[MAX_KEYS]; // 1, 2, 4 or 8 bytes
	uint32_t key_shift[MAX_KEYS]; // bit position inside the (single) packed key word
};

// Non-zero when the 8-byte integer x is too large for the 64-bit per-thread partials of FASTREG / PRIV / WPRIV and
// must take the global path: x outside [-2^40, 2^40) for a signed input, x >= 2^40 for an unsigned one.  The signed
// test alone, (x + 2^40) >> 41, would let an unsigned x >= 2^64 - 2^40 wrap to a small value and stay.  Both tests
// only read the high word (adding 2^40 leaves the low word alone): signed (hi + 2^8) >> 9, unsigned hi >> 8.
// With them, a partial of k kept values lies in (-k 2^40, k 2^40), inside the signed 64-bit range for k < 2^23, so
// the reductions may widen every partial as a SIGNED 64-bit value, unsigned inputs included.
__device__ __forceinline__ uint32_t reg_value_too_big(uint64_t x, bool is_unsigned) {
	const uint32_t bias = is_unsigned ? 0u : 1u << 8;
	const uint32_t mask = is_unsigned ? ~0xffu : ~0x1ffu;
	return ((uint32_t)(x >> 32) + bias) & mask;
}

// zero-extended load of a 1/2/4/8-byte integer from a staged tile
__device__ __forceinline__ uint64_t stage_load_uint(const unsigned char *p, uint32_t width) {
	if (width == 8) {
		return *(const uint64_t *)p;
	}
	// 1, 2 or 4 bytes: one aligned 32-bit load + shift + mask, branch-free
	uint32_t a = (uint32_t)(uintptr_t)p;
	uint32_t word = *(const uint32_t *)(p - (a & 3));
	uint32_t v = word >> ((a & 3) * 8);
	return width == 4 ? v : (v & ((1u << (width * 8)) - 1));
}

