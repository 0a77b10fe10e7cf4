// K4 join_probe, TMA-staged variant (the fast path of b200_join_probe).
//
// Eligibility: one key column (exact keys), every probe column FLAT and 16-byte aligned.  Each CTA walks 1024-row
// tiles of the probe batch: the key column and the lhs pass-through columns are bulk-copied HBM -> shared memory
// by TMA (tile_pipe.cuh) two stages ahead; each thread then owns 4 rows of the tile and
//   1. issues the 4 table-slot loads (one 16-byte __ldg each: key + head row + inline payload) back to back, so
//      4 independent random HBM accesses are in flight per thread,
//   2. resolves collisions (linear probing, rare), counts result rows,
//   3. claims output positions: warp scan -> one shared-memory atomic per warp -> ONE global atomic per tile,
//   4. writes the result rows (lhs values straight from the staged tile, payload from the slot / payload store).
// Reference semantics: see join.cu.
#include "join.cuh"
#include "tile_pipe.cuh"
#include <cstring>
#include <cstdlib>

#define JT_THREADS 256
#define JT_TILE 1024
#define JT_ROWS (JT_TILE / JT_THREADS)
#define JT_STAGES 3

struct ProbeTileArgs {
	JoinView J;
	TileCols tc;
	int key_col, key_valid_col; // tile column indices
	int key_type;
	int nlhs;
	int lhs_col[MAX_LHS], lhs_valid_col[MAX_LHS];
	int lhs_width[MAX_LHS];
	int pay_width[2];
	ProbeOut po;
	int join_type;
	uint64_t n;
	uint64_t out_capacity;
	unsigned long long *counters;
	int stages;
};

__device__ __forceinline__ void copy_value(void *dst, uint64_t opos, const unsigned char *src, int width) {
	switch (width) {
	case 1:
		((uint8_t *)dst)[opos] = *src;
		break;
	case 2:
		((uint16_t *)dst)[opos] = *(const uint16_t *)src;
		break;
	case 4:
		((uint32_t *)dst)[opos] = *(const uint32_t *)src;
		break;
	default:
		((uint64_t *)dst)[opos] = *(const uint64_t *)src;
		break;
	}
}

template <bool FAST8>
__device__ __forceinline__ void emit_tile_row(const ProbeTileArgs &A, const unsigned char *stage, uint32_t r,
                                              uint64_t prow, uint64_t opos, uint32_t brow, uint32_t inl,
                                              bool with_payload) {
	const ProbeOut &po = A.po;
	const JoinView &J = A.J;
	if (po.lhs_sel) {
		po.lhs_sel[opos] = (uint32_t)prow;
	}
	if (FAST8) {
		// every lhs column is 8 bytes wide without NULLs: straight 64-bit copies
#pragma unroll
		for (int j = 0; j < 4; j++) {
			if (j < A.nlhs) {
				((uint64_t *)po.lhs_data[j])[opos] =
				    *(const uint64_t *)(stage + A.tc.c[A.lhs_col[j]].smem_off + (size_t)r * 8);
			}
		}
	}
	for (int j = 0; j < (FAST8 ? 0 : A.nlhs); j++) {
		int w = A.lhs_width[j];
		copy_value(po.lhs_data[j], opos, stage + A.tc.c[A.lhs_col[j]].smem_off + (size_t)r * w, w);
		if (po.lhs_valid[j] && A.lhs_valid_col[j] >= 0 &&
		    !((stage[A.tc.c[A.lhs_valid_col[j]].smem_off + (r >> 3)] >> (r & 7)) & 1)) {
			atomicAnd((unsigned long long *)&po.lhs_valid[j][opos >> 6], ~(1ULL << (opos & 63)));
		}
	}
	if (!with_payload) {
		return;
	}
	if (brow == ROW_NONE) {
		for (int p = 0; p < J.ps.n; p++) {
			store_raw(po.pay_data[p], J.ps.type[p], opos, 0);
			atomicAnd((unsigned long long *)&po.pay_valid[p][opos >> 6], ~(1ULL << (opos & 63)));
		}
		return;
	}
	if (J.inline_payload) {
		int sh = 0;
		for (int p = 0; p < J.ps.n; p++) {
			int sz = b200_type_size(J.ps.type[p]);
			uint32_t bits = inl >> sh;
			sh += sz * 8;
			store_raw(po.pay_data[p], J.ps.type[p], opos, (uint64_t)bits); // store_raw truncates to the type width
		}
		return;
	}
	for (int p = 0; p < J.ps.n; p++) {
		DCol c;
		c.data = J.ps.data[p];
		c.type = J.ps.type[p];
		c.sel = nullptr;
		c.validity = J.ps.validity[p];
		c.vtype = B200_FLAT_VECTOR;
		store_raw(po.pay_data[p], c.type, opos, col_load_raw(c, brow));
		if (po.pay_valid[p] && !col_valid_at(c, brow)) {
			atomicAnd((unsigned long long *)&po.pay_valid[p][opos >> 6], ~(1ULL << (opos & 63)));
		}
	}
}

template <bool FAST8, bool LEAN>
__global__ void __launch_bounds__(JT_THREADS, 2) join_probe_tile_kernel(const __grid_constant__ ProbeTileArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * JT_STAGES];
	__shared__ unsigned int tile_cursor;
	__shared__ unsigned long long tile_base;
	const JoinView &J = A.J;
	const int tid = threadIdx.x, lane = tid & 31;
	const int jt = A.join_type;
	const bool with_payload = jt == B200_JOIN_INNER || jt == B200_JOIN_LEFT;
	if (tid == 0) {
		tile_cursor = 0;
	}
	const TileCol kc = A.tc.c[A.key_col];
	const int kwidth = b200_type_size(A.key_type);

	tp_tile_loop_sync(A.tc, A.stages, smem_raw, bars, 0, A.n, [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		if constexpr (LEAN) {
			// INNER join, unique build keys, 8-byte integer key and lhs columns, payload inline in the table entry
			// (or none): the shape of a PK-FK join such as TPC-H Q14.  No per-row switches, one table load per row.
			uint64_t lkey[JT_ROWS];
			uint32_t ent[JT_ROWS], lpos[JT_ROWS];
			bool hit[JT_ROWS];
#pragma unroll
			for (int k = 0; k < JT_ROWS; k++) {
				uint32_t r = k * JT_THREADS + tid;
				ent[k] = 0;
				hit[k] = false;
				if (r < rows_in_tile) {
					lkey[k] = *(const uint64_t *)(stage + kc.smem_off + (size_t)r * 8);
					if (J.dense) {
						uint64_t idx = lkey[k] - J.dense_min;
						if (idx < J.dense_range) {
							ent[k] = __ldg(&J.dense[idx]);
						}
						hit[k] = ent[k] != 0;
						ent[k] >>= 8;
					}
				}
			}
			if (!J.dense) {
				// open-addressing table: issue the 4 first slot loads back to back, then resolve (linear probing)
				uint64_t sl[JT_ROWS];
				uint4 v[JT_ROWS];
				bool pend[JT_ROWS];
#pragma unroll
				for (int k = 0; k < JT_ROWS; k++) {
					uint32_t r = k * JT_THREADS + tid;
					pend[k] = false;
					if (r < rows_in_tile && !J.build_empty) {
						if (lkey[k] == EMPTY_KEY) {
							const JoinSlot &s = J.slots[J.mask + 1];
							hit[k] = s.head != ROW_NONE;
							ent[k] = s.inl;
						} else {
							sl[k] = murmur64(lkey[k]) & J.mask;
							v[k] = __ldg((const uint4 *)&J.slots[sl[k]]);
							pend[k] = true;
						}
					}
				}
#pragma unroll
				for (int k = 0; k < JT_ROWS; k++) {
					while (pend[k]) {
						uint64_t sk = ((uint64_t)v[k].y << 32) | v[k].x;
						if (sk == lkey[k]) {
							hit[k] = true;
							ent[k] = v[k].w;
							pend[k] = false;
						} else if (sk == EMPTY_KEY) {
							pend[k] = false;
						} else {
							sl[k] = (sl[k] + 1) & J.mask;
							v[k] = __ldg((const uint4 *)&J.slots[sl[k]]);
						}
					}
				}
			}
#pragma unroll
			for (int k = 0; k < JT_ROWS; k++) {
				uint32_t m = __ballot_sync(0xffffffffu, hit[k]);
				uint32_t wbase = 0;
				if (lane == 0 && m) {
					wbase = atomicAdd(&tile_cursor, __popc(m));
				}
				wbase = __shfl_sync(0xffffffffu, wbase, 0);
				lpos[k] = wbase + __popc(m & ((1u << lane) - 1));
			}
			__syncthreads();
			if (tid == 0) {
				tile_base = tile_cursor ? atomicAdd(&A.counters[1], (unsigned long long)tile_cursor) : 0ULL;
				tile_cursor = 0;
			}
			__syncthreads();
			const unsigned long long lbase = tile_base;
#pragma unroll
			for (int k = 0; k < JT_ROWS; k++) {
				if (!hit[k]) {
					continue;
				}
				uint32_t r = k * JT_THREADS + tid;
				uint64_t opos = lbase + lpos[k];
				if (opos >= A.out_capacity) {
					continue;
				}
				if (A.po.lhs_sel) {
					A.po.lhs_sel[opos] = (uint32_t)(row0 + r);
				}
#pragma unroll
				for (int j = 0; j < 4; j++) {
					if (j < A.nlhs) {
						__stcs((unsigned long long *)A.po.lhs_data[j] + opos,
						       *(const unsigned long long *)(stage + A.tc.c[A.lhs_col[j]].smem_off + (size_t)r * 8));
					}
				}
				// inline payload: <= 2 columns of 1 or 2 bytes packed in the entry
				uint32_t bits = ent[k];
#pragma unroll
				for (int p = 0; p < 2; p++) {
					if (p < J.ps.n) {
						if (A.pay_width[p] == 1) {
							((uint8_t *)A.po.pay_data[p])[opos] = (uint8_t)bits;
							bits >>= 8;
						} else {
							((uint16_t *)A.po.pay_data[p])[opos] = (uint16_t)bits;
							bits >>= 16;
						}
					}
				}
			}
			return;
		}
		uint64_t key[JT_ROWS];
		uint64_t slot[JT_ROWS];
		uint4 sv[JT_ROWS];
		uint32_t first[JT_ROWS], inl[JT_ROWS], cnt[JT_ROWS], opos_local[JT_ROWS];
		bool knull[JT_ROWS], pending[JT_ROWS];
		// 1. keys and the first slot load of every row
#pragma unroll
		for (int k = 0; k < JT_ROWS; k++) {
			uint32_t r = k * JT_THREADS + tid;
			first[k] = ROW_NONE;
			inl[k] = 0;
			knull[k] = false;
			pending[k] = false;
			if (r < rows_in_tile) {
				if (FAST8) {
					key[k] = *(const uint64_t *)(stage + kc.smem_off + (size_t)r * 8); // 8-byte integer key, no NULLs
				} else {
					DCol d;
					d.data = stage + kc.smem_off;
					d.sel = nullptr;
					d.validity = nullptr;
					d.type = A.key_type;
					d.vtype = B200_FLAT_VECTOR;
					key[k] = canonical_key_bits(A.key_type, col_load_raw(d, r));
					if (A.key_valid_col >= 0) {
						knull[k] = !((stage[A.tc.c[A.key_valid_col].smem_off + (r >> 3)] >> (r & 7)) & 1);
					}
				}
				if (!knull[k] && !J.build_empty && J.dense) {
					// direct-addressed table: one 4-byte load; L2-resident while it fits (50 MB of L2 on an H100 =
					// ~12 M keys; SF100's 20 M-key part table, 80 MB, is served partly from HBM)
					uint64_t idx = key[k] - J.dense_min;
					if (idx < J.dense_range) {
						uint32_t e = __ldg(&J.dense[idx]);
						if (e) {
							inl[k] = e >> 8;
							first[k] = J.inline_payload ? 0u : e - 1;
						}
					}
				} else if (!knull[k] && !J.build_empty) {
					if (key[k] == EMPTY_KEY) {
						const JoinSlot &s = J.slots[J.mask + 1];
						first[k] = s.head;
						inl[k] = s.inl;
					} else {
						slot[k] = (FAST8 ? murmur64(key[k]) : hash_raw(A.key_type, key[k])) & J.mask;
						sv[k] = __ldg((const uint4 *)&J.slots[slot[k]]);
						pending[k] = true;
					}
				}
			}
		}
		(void)kwidth;
		// 2. resolve (linear probing)
#pragma unroll
		for (int k = 0; k < JT_ROWS; k++) {
			while (pending[k]) {
				uint64_t sk = ((uint64_t)sv[k].y << 32) | sv[k].x;
				if (sk == key[k]) {
					first[k] = sv[k].z;
					inl[k] = sv[k].w;
					pending[k] = false;
				} else if (sk == EMPTY_KEY) {
					pending[k] = false;
				} else {
					slot[k] = (slot[k] + 1) & J.mask;
					sv[k] = __ldg((const uint4 *)&J.slots[slot[k]]);
				}
			}
		}
		// 3. result rows per probe row
#pragma unroll
		for (int k = 0; k < JT_ROWS; k++) {
			uint32_t r = k * JT_THREADS + tid;
			uint32_t c = 0;
			if (r < rows_in_tile) {
				switch (jt) {
				case B200_JOIN_INNER:
				case B200_JOIN_LEFT:
					if (first[k] != ROW_NONE) {
						if (J.unique) {
							c = 1;
						} else {
							for (uint32_t b = first[k]; b != ROW_NONE; b = J.next[b]) {
								c++;
							}
						}
					} else if (jt == B200_JOIN_LEFT) {
						c = 1;
					}
					break;
				case B200_JOIN_SEMI:
					c = first[k] != ROW_NONE;
					break;
				case B200_JOIN_ANTI:
					c = first[k] == ROW_NONE;
					break;
				default:
					c = 1;
					break;
				}
			}
			cnt[k] = c;
			// warp scan + one shared atomic per warp
			uint32_t incl = c;
#pragma unroll
			for (int off = 1; off < 32; off <<= 1) {
				uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
				if (lane >= off) {
					incl += t;
				}
			}
			uint32_t wtotal = __shfl_sync(0xffffffffu, incl, 31);
			uint32_t wbase = 0;
			if (lane == 0 && wtotal) {
				wbase = atomicAdd(&tile_cursor, wtotal);
			}
			wbase = __shfl_sync(0xffffffffu, wbase, 0);
			opos_local[k] = wbase + incl - c;
		}
		__syncthreads();
		if (tid == 0) {
			tile_base = tile_cursor ? atomicAdd(&A.counters[1], (unsigned long long)tile_cursor) : 0ULL;
			tile_cursor = 0;
		}
		__syncthreads();
		const unsigned long long base = tile_base;
		// 4. write
#pragma unroll
		for (int k = 0; k < JT_ROWS; k++) {
			if (!cnt[k]) {
				continue;
			}
			uint32_t r = k * JT_THREADS + tid;
			uint64_t opos = base + opos_local[k];
			if (opos + cnt[k] > A.out_capacity) {
				continue; // the host sees cursor > capacity and reports B200_ERR_CAPACITY
			}
			uint64_t prow = row0 + r;
			switch (jt) {
			case B200_JOIN_INNER:
			case B200_JOIN_LEFT:
				if (first[k] == ROW_NONE || J.unique) {
					if (J.matched && first[k] != ROW_NONE) {
						J.matched[first[k]] = 1;
					}
					emit_tile_row<FAST8>(A, stage, r, prow, opos, first[k], inl[k], true);
				} else {
					for (uint32_t b = first[k]; b != ROW_NONE; b = J.next[b]) {
						if (J.matched) {
							J.matched[b] = 1;
						}
						emit_tile_row<FAST8>(A, stage, r, prow, opos++, b, inl[k], true);
					}
				}
				break;
			case B200_JOIN_SEMI:
			case B200_JOIN_ANTI:
				emit_tile_row<FAST8>(A, stage, r, prow, opos, ROW_NONE, 0, false);
				break;
			default: {
				emit_tile_row<FAST8>(A, stage, r, prow, opos, ROW_NONE, 0, false);
				bool matched = first[k] != ROW_NONE;
				A.po.mark[opos] = matched ? 1 : 0;
				if (!matched && (knull[k] || J.build_has_null) && !J.build_empty) {
					atomicAnd((unsigned long long *)&A.po.mark_valid[opos >> 6], ~(1ULL << (opos & 63)));
				}
				break;
			}
			}
		}
		(void)with_payload;
	});
}

// ------------------------------------------------------------------ LEAN2: the PK-FK probe, instruction-lean
// Same contract as join_probe_tile_kernel<true, true> (INNER join, unique build keys, 8-byte key and lhs columns
// without NULLs, payload inline in the table entry or none), written so that nothing is re-derived per row: column
// offsets, output pointers and payload widths are template / register constants, the four (or eight) table loads of a
// thread are issued back to back, result positions come from one ballot per row slice and ONE shared-memory atomic
// per warp per tile, so that the kernel is bound by memory rather than by instruction issue.
template <int NLHS, int ROWS, bool DENSE>
__global__ void __launch_bounds__(JT_THREADS, 2) join_probe_lean2_kernel(const __grid_constant__ ProbeTileArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * JT_STAGES];
	__shared__ unsigned int tile_cursor;
	__shared__ unsigned long long tile_base;
	const int tid = threadIdx.x, lane = tid & 31;
	const uint32_t key_off = A.tc.c[A.key_col].smem_off;
	uint32_t lhs_off[NLHS > 0 ? NLHS : 1];
	unsigned long long *lhs_out[NLHS > 0 ? NLHS : 1];
#pragma unroll
	for (int j = 0; j < NLHS; j++) {
		lhs_off[j] = A.tc.c[A.lhs_col[j]].smem_off;
		lhs_out[j] = (unsigned long long *)A.po.lhs_data[j];
	}
	const int npay = A.J.ps.n;
	const int pw0 = A.pay_width[0], pw1 = A.pay_width[1];
	uint8_t *const pay0 = (uint8_t *)A.po.pay_data[0];
	uint8_t *const pay1 = (uint8_t *)A.po.pay_data[1];
	uint32_t *const lhs_sel = A.po.lhs_sel;
	const uint32_t *const dense = A.J.dense;
	const uint64_t dmin = A.J.dense_min, drange = A.J.dense_range;
	const JoinSlot *const slots = A.J.slots;
	const uint64_t mask = A.J.mask;
	const bool build_empty = A.J.build_empty;
	const uint64_t out_capacity = A.out_capacity;
	if (tid == 0) {
		tile_cursor = 0;
	}
	tp_tile_loop_sync(A.tc, A.stages, smem_raw, bars, 0, A.n, [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		const uint64_t *kcol = (const uint64_t *)(stage + key_off);
		uint32_t ent[ROWS];
		bool hit[ROWS];
		if (DENSE) {
#pragma unroll
			for (int k = 0; k < ROWS; k++) {
				uint32_t r = k * JT_THREADS + tid;
				ent[k] = 0;
				if (r < rows_in_tile) {
					uint64_t idx = kcol[r] - dmin;
					if (idx < drange) {
						ent[k] = __ldg(&dense[idx]);
					}
				}
			}
#pragma unroll
			for (int k = 0; k < ROWS; k++) {
				hit[k] = ent[k] != 0;
				ent[k] >>= 8;
			}
		} else {
			uint64_t key[ROWS], sl[ROWS];
			uint4 v[ROWS];
			bool pend[ROWS];
#pragma unroll
			for (int k = 0; k < ROWS; k++) {
				uint32_t r = k * JT_THREADS + tid;
				pend[k] = false;
				hit[k] = false;
				ent[k] = 0;
				if (r < rows_in_tile && !build_empty) {
					key[k] = kcol[r];
					if (key[k] == EMPTY_KEY) {
						const JoinSlot &s = slots[mask + 1];
						hit[k] = s.head != ROW_NONE;
						ent[k] = s.inl;
					} else {
						sl[k] = murmur64(key[k]) & mask;
						v[k] = __ldg((const uint4 *)&slots[sl[k]]);
						pend[k] = true;
					}
				}
			}
#pragma unroll
			for (int k = 0; k < ROWS; k++) {
				while (pend[k]) {
					uint64_t sk = ((uint64_t)v[k].y << 32) | v[k].x;
					if (sk == key[k]) {
						hit[k] = true;
						ent[k] = v[k].w;
						pend[k] = false;
					} else if (sk == EMPTY_KEY) {
						pend[k] = false;
					} else {
						sl[k] = (sl[k] + 1) & mask;
						v[k] = __ldg((const uint4 *)&slots[sl[k]]);
					}
				}
			}
		}
		// output positions: one ballot per row slice, one shared atomic per warp
		uint32_t lpos[ROWS];
		uint32_t wtotal = 0;
#pragma unroll
		for (int k = 0; k < ROWS; k++) {
			uint32_t m = __ballot_sync(0xffffffffu, hit[k]);
			lpos[k] = wtotal + __popc(m & ((1u << lane) - 1));
			wtotal += __popc(m);
		}
		uint32_t wbase = 0;
		if (lane == 0 && wtotal) {
			wbase = atomicAdd(&tile_cursor, wtotal);
		}
		wbase = __shfl_sync(0xffffffffu, wbase, 0);
		__syncthreads();
		if (tid == 0) {
			tile_base = tile_cursor ? atomicAdd(&A.counters[1], (unsigned long long)tile_cursor) : 0ULL;
			tile_cursor = 0;
		}
		__syncthreads();
		const uint64_t obase = tile_base + wbase;
#pragma unroll
		for (int k = 0; k < ROWS; k++) {
			if (!hit[k]) {
				continue;
			}
			uint32_t r = k * JT_THREADS + tid;
			uint64_t opos = obase + lpos[k];
			if (opos >= out_capacity) {
				continue;
			}
			if (lhs_sel) {
				lhs_sel[opos] = (uint32_t)(row0 + r);
			}
#pragma unroll
			for (int j = 0; j < NLHS; j++) {
				__stcs(lhs_out[j] + opos, *(const unsigned long long *)(stage + lhs_off[j] + (size_t)r * 8));
			}
			if (npay > 0) {
				uint32_t bits = ent[k];
				if (pw0 == 1) {
					pay0[opos] = (uint8_t)bits;
					bits >>= 8;
				} else {
					((uint16_t *)pay0)[opos] = (uint16_t)bits;
					bits >>= 16;
				}
				if (npay > 1) {
					if (pw1 == 1) {
						pay1[opos] = (uint8_t)bits;
					} else {
						((uint16_t *)pay1)[opos] = (uint16_t)bits;
					}
				}
			}
		}
	});
}

template <int ROWS, bool DENSE>
static int launch_lean2(b200_ctx *ctx, const ProbeTileArgs &A, unsigned grid, size_t smem) {
#define LEAN2_CASE(N)                                                                                                  \
	case N: {                                                                                                          \
		static bool attr_set = false;                                                                                  \
		if (!attr_set) {                                                                                               \
			CUDA_TRY(cudaFuncSetAttribute(join_probe_lean2_kernel<N, ROWS, DENSE>,                                     \
			                              cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));                   \
			attr_set = true;                                                                                           \
		}                                                                                                              \
		join_probe_lean2_kernel<N, ROWS, DENSE><<<grid, JT_THREADS, smem, ctx->stream>>>(A);                           \
		return B200_OK;                                                                                                \
	}
	switch (A.nlhs) {
		LEAN2_CASE(0)
		LEAN2_CASE(1)
		LEAN2_CASE(2)
		LEAN2_CASE(3)
		LEAN2_CASE(4)
	}
#undef LEAN2_CASE
	return B200_ERR_INVALID;
}

// host: returns B200_OK when the launch was made, B200_ERR_INVALID when the batch is not eligible
int b200_join_probe_tile(b200_ctx *ctx, const JoinView &J, const KeyCols &keys, const ProbeOut &po, int join_type,
                         uint64_t n, uint64_t out_capacity, unsigned long long *counters) {
	if (!J.exact || keys.n != 1 || n == 0) {
		return B200_ERR_INVALID;
	}
	ProbeTileArgs A;
	memset(&A, 0, sizeof(A));
	A.J = J;
	A.po = po;
	A.join_type = join_type;
	A.n = n;
	A.out_capacity = out_capacity;
	A.counters = counters;
	A.key_type = keys.c[0].type;
	A.nlhs = po.nlhs;
	auto add = [&](const void *ptr, uint32_t width) -> int {
		for (int i = 0; i < A.tc.n; i++) {
			if (A.tc.c[i].ptr == (const unsigned char *)ptr && A.tc.c[i].width == width) {
				return i;
			}
		}
		if (A.tc.n >= TP_MAX_COLS) {
			return -1;
		}
		A.tc.c[A.tc.n].ptr = (const unsigned char *)ptr;
		A.tc.c[A.tc.n].width = width;
		return A.tc.n++;
	};
	auto stageable = [](const DCol &c) {
		return c.vtype == B200_FLAT_VECTOR && tile_ptr_ok(c.data) && (!c.validity || tile_ptr_ok(c.validity));
	};
	if (!stageable(keys.c[0])) {
		return B200_ERR_INVALID;
	}
	A.key_col = add(keys.c[0].data, b200_type_size(keys.c[0].type));
	A.key_valid_col = keys.c[0].validity ? add(keys.c[0].validity, 0) : -1;
	for (int j = 0; j < po.nlhs; j++) {
		const DCol &c = po.lhs_src[j];
		if (!stageable(c)) {
			return B200_ERR_INVALID;
		}
		A.lhs_width[j] = b200_type_size(c.type);
		A.lhs_col[j] = add(c.data, A.lhs_width[j]);
		A.lhs_valid_col[j] = c.validity ? add(c.validity, 0) : -1;
		if (A.lhs_col[j] < 0 || (c.validity && A.lhs_valid_col[j] < 0)) {
			return B200_ERR_INVALID;
		}
	}
	if (A.key_col < 0 || (keys.c[0].validity && A.key_valid_col < 0)) {
		return B200_ERR_INVALID;
	}
	tile_cols_finish(&A.tc, JT_TILE);
	// two CTAs per SM: <= ~110 KB of stages each
	A.stages = JT_STAGES;
	{
		const char *env = getenv("B200_JOIN_STAGES"); // experiment knob
		if (env && (atoi(env) == 2 || atoi(env) == 3)) {
			A.stages = atoi(env);
		}
	}
	while (A.stages > 2 && (size_t)A.stages * A.tc.stage_bytes > 108 * 1024) {
		A.stages--;
	}
	size_t smem = (size_t)A.stages * A.tc.stage_bytes;
	if (smem > 220 * 1024) {
		return B200_ERR_INVALID;
	}
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(join_probe_tile_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
		                              220 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(join_probe_tile_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
		                              220 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(join_probe_tile_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
		                              220 * 1024));
		attr_set = true;
	}
	// flagship shape (TPC-H keys are BIGINT, DECIMAL(15,2) payloads are int64): specialised loads / copies
	bool fast8 = (A.key_type == B200_INT64 || A.key_type == B200_UINT64) && A.key_valid_col < 0 && A.nlhs <= 4;
	for (int j = 0; j < A.nlhs; j++) {
		fast8 = fast8 && A.lhs_width[j] == 8 && A.lhs_valid_col[j] < 0;
	}
	uint64_t ntiles = (n + JT_TILE - 1) / JT_TILE;
	int per_sm = (int)((220 * 1024) / (smem + 1024));
	per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
	uint64_t max_grid = (uint64_t)ctx->sm_count * per_sm;
	uint64_t grid = ntiles < max_grid ? ntiles : max_grid;
	// lean path: INNER join on unique keys whose payload (if any) is inline in the table entry.  Neither lean kernel
	// tracks build rows, so a RIGHT join (probed as INNER, with match flags) never takes it.
	bool lean = fast8 && join_type == B200_JOIN_INNER && !J.matched && J.unique && (J.ps.n == 0 || J.inline_payload) &&
	            J.ps.n <= 2;
	for (int p = 0; p < J.ps.n && p < 2; p++) {
		A.pay_width[p] = b200_type_size(J.ps.type[p]);
		lean = lean && A.pay_width[p] <= 2 && !po.pay_valid[p];
	}
	if (lean && !getenv("B200_JOIN_LEAN1")) {
		// LEAN2: 8 rows per thread (2048-row tiles, 2 stages) unless B200_JOIN_ROWS=4
		const char *renv = getenv("B200_JOIN_ROWS");
		int rows = renv && atoi(renv) == 4 ? 4 : 8;
		tile_cols_finish(&A.tc, (uint32_t)rows * JT_THREADS);
		A.stages = rows == 8 ? 2 : 3;
		size_t smem2 = (size_t)A.stages * A.tc.stage_bytes;
		if (smem2 <= 110 * 1024) {
			uint64_t ntiles2 = (n + A.tc.tile_rows - 1) / A.tc.tile_rows;
			uint64_t mg = (uint64_t)ctx->sm_count * 2;
			unsigned g2 = (unsigned)(ntiles2 < mg ? ntiles2 : mg);
			int rc2 = rows == 8 ? (J.dense ? launch_lean2<8, true>(ctx, A, g2, smem2) : launch_lean2<8, false>(ctx, A, g2, smem2))
			                    : (J.dense ? launch_lean2<4, true>(ctx, A, g2, smem2) : launch_lean2<4, false>(ctx, A, g2, smem2));
			B200_TRY(rc2);
			ctx->launches++;
			CUDA_TRY(cudaGetLastError());
			return B200_OK;
		}
		tile_cols_finish(&A.tc, JT_TILE);
		A.stages = JT_STAGES;
		while (A.stages > 2 && (size_t)A.stages * A.tc.stage_bytes > 108 * 1024) {
			A.stages--;
		}
	}
	if (lean) {
		join_probe_tile_kernel<true, true><<<(unsigned)grid, JT_THREADS, smem, ctx->stream>>>(A);
	} else if (fast8) {
		join_probe_tile_kernel<true, false><<<(unsigned)grid, JT_THREADS, smem, ctx->stream>>>(A);
	} else {
		join_probe_tile_kernel<false, false><<<(unsigned)grid, JT_THREADS, smem, ctx->stream>>>(A);
	}
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}
