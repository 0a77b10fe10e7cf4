// K6 sink path PRIV: thread-private accumulators in shared memory for ~9..64 groups (SSB Q4.1: 35 groups).
//
// Why not shared-memory atomics (MID): a shared-memory atomic is serviced per LANE, so a row with S sums pays for
// 1 + 4 S lane-serialised updates per SM, while plain LDS / STS move 128 B per cycle.  So, like the register path (FASTREG) but with the
// states in shared memory: every consumer thread owns a private copy of the state of every slot, laid out
// [slot][sum][thread] (a warp's accesses hit 32 consecutive 8-byte words: conflict free).  A row costs one lookup in
// a small CTA-wide directory (packed key -> slot) and, per sum, LDS.64 + IADD.64 + STS.64.  No atomics, no shuffles
// on the row path.  The private copies are reduced in 128-bit at the end of the kernel and merged into the global
// table with one atomic per (CTA, group, state), exactly like FAST / FASTREG.
//
// Eligibility (same as FASTREG): integer group keys without NULLs packed in <= 7 bytes, every aggregate is
// sum / avg / count over non-NULL 8-byte integers.  Values outside [-2^40, 2^40) (unsigned: >= 2^40, see
// reg_value_too_big) and keys beyond the CTA's slots take the global path inline (row_to_global); rows whose key missed
// are counted in counters[1].
// Reference semantics: GroupedAggregateHashTable::FindOrCreateGroupsInternal + UpdateAggregates
// (src/execution/aggregate_hashtable.cpp:803-977,688-722), integer sums as hugeint (sum_helpers.hpp:155-215).
#include "agg_tile.cuh"
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include <vector>

#define PRIV_DIR_CAP 1024 // directory entries (power of two); at most PRIV_DIR_LIMIT + resident threads are ever used
#define PRIV_DIR_LIMIT 256
#define PRIV_RB 4 // rows per thread in flight
#define PRIV_KEYMASK ((1ULL << 56) - 1)
#define PRIV_LOCKED 0xffULL
#define PRIV_OVERFLOW 0xfeULL

struct PrivShared {
	unsigned long long dir[PRIV_DIR_CAP]; // key56 | (slot + 1) << 56 ; tag 0xff = being inserted, 0xfe = no slot left
	unsigned int nentries;                // directory entries (incl. overflow entries)
};

// slot of `key56` in the CTA's directory, -1 when the key has no private slot (-> global path)
__device__ __forceinline__ int priv_lookup(PrivShared &S, unsigned long long *slot_key, int nslots, unsigned long long key56) {
	uint32_t pos = (uint32_t)((key56 * 0x9E3779B97F4A7C15ULL) >> 44) & (PRIV_DIR_CAP - 1);
	while (true) {
		unsigned long long e = *(volatile unsigned long long *)&S.dir[pos];
		if (e == 0ULL) {
			if (*(volatile unsigned int *)&S.nentries >= PRIV_DIR_LIMIT) {
				return -1;
			}
			unsigned long long old = atomicCAS(&S.dir[pos], 0ULL, key56 | (PRIV_LOCKED << 56));
			if (old == 0ULL) {
				unsigned int s = atomicAdd(&S.nentries, 1u);
				unsigned long long tag = PRIV_OVERFLOW;
				if ((int)s < nslots) {
					slot_key[s] = key56 | (1ULL << 56);
					tag = s + 1;
				}
				__threadfence_block();
				*(volatile unsigned long long *)&S.dir[pos] = key56 | (tag << 56);
				return tag == PRIV_OVERFLOW ? -1 : (int)s;
			}
			e = old;
		}
		if ((e & PRIV_KEYMASK) == key56) {
			unsigned long long tag = e >> 56;
			while (tag == PRIV_LOCKED) {
				tag = *(volatile unsigned long long *)&S.dir[pos] >> 56;
			}
			return tag == PRIV_OVERFLOW ? -1 : (int)tag - 1;
		}
		pos = (pos + 1) & (PRIV_DIR_CAP - 1);
	}
}

// DIRECT addressing, one key column of width sizeof(T), PRIV_RB rows: slot += lut[value - min] * stride.  The width
// dispatch sits OUTSIDE the row loop (decoding the key per row with run-time widths costs more instructions than the
// rest of the row's work).
template <class T>
__device__ __forceinline__ void direct_codes(const unsigned char *col, const uint8_t *lut, uint64_t kmin64, uint32_t range,
                                             uint32_t stride, const uint32_t (&row)[PRIV_RB], int (&sl)[PRIV_RB],
                                             bool (&ok)[PRIV_RB]) {
	const T *p = (const T *)col;
	const T kmin = (T)kmin64;
#pragma unroll
	for (int k = 0; k < PRIV_RB; k++) {
		const T d = (T)(p[row[k]] - kmin); // wrap-around: values below the minimum become huge
		const bool in = (uint64_t)d < (uint64_t)range;
		const uint32_t c = lut[in ? (uint32_t)d : 0u];
		ok[k] = ok[k] && in && c != 0xffu;
		sl[k] += (int)(c * stride);
	}
}

// KW: 1 = every key column is one byte (Q1), 4 = one 4-byte key, 0 = generic key descriptors, 2 = DIRECT addressing
template <int NSUM, int KW>
__global__ void __launch_bounds__(512 + 32, 1)
    agg_priv_kernel(const __grid_constant__ TileArgs A, const __grid_constant__ RegLayout R, int SLOTS, int NC,
                    const __grid_constant__ PrivDirect PD) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ PrivShared S;
	__shared__ uint64_t bars[2 * AT_MAX_STAGES];
	const int tid = threadIdx.x;
	const AggLayout &L = A.L;
	// [slot][sum][thread] 64-bit partial sums, [slot][thread] 32-bit row counts, slot keys, then the stage ring
	uint64_t *acc = (uint64_t *)smem_raw;
	uint32_t *rowc = (uint32_t *)(acc + (size_t)SLOTS * NSUM * NC);
	unsigned long long *slot_key = (unsigned long long *)(rowc + (size_t)SLOTS * NC);
	size_t state_bytes = (size_t)SLOTS * NSUM * NC * 8 + (size_t)SLOTS * NC * 4 + (size_t)SLOTS * 8;
	uint8_t *lut = smem_raw + ((state_bytes + 15) & ~(size_t)15);
	if (KW == 2) {
		state_bytes = ((state_bytes + 15) & ~(size_t)15) + PD.lut_bytes;
	}
	unsigned char *stages = smem_raw + ((state_bytes + 127) & ~(size_t)127);

	for (int i = tid; i < PRIV_DIR_CAP; i += blockDim.x) {
		S.dir[i] = 0ULL;
	}
	if (tid == 0) {
		S.nentries = 0;
	}
	if (tid < NC) {
		for (int s = 0; s < SLOTS; s++) {
#pragma unroll
			for (int j = 0; j < NSUM; j++) {
				acc[((size_t)s * NSUM + j) * NC + tid] = 0;
			}
			rowc[(size_t)s * NC + tid] = 0;
		}
	}
	for (int s = tid; s < SLOTS; s += blockDim.x) {
		slot_key[s] = KW == 2 ? PD.slot_keys[s] : 0ULL;
	}
	if (KW == 2) {
		for (uint32_t i = tid; i < PD.lut_bytes; i += blockDim.x) {
			lut[i] = PD.lut[i];
		}
	}
	unsigned long long missed = 0;
	__syncthreads();

	tp_tile_loop(A.tc, A.stages, stages, bars, A.row_begin, A.row_end, NC,
	             [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		for (uint32_t rb = tid; rb < rows_in_tile; rb += PRIV_RB * NC) {
			// 1. keys, values and directory lookups of up to PRIV_RB rows (independent shared-memory loads in flight)
			unsigned long long key[PRIV_RB];
			uint64_t x[PRIV_RB][NSUM];
			int slot[PRIV_RB];
			bool live[PRIV_RB];
			if constexpr (KW == 2) {
				uint32_t row[PRIV_RB];
				int sl[PRIV_RB];
				bool ok[PRIV_RB];
#pragma unroll
				for (int k = 0; k < PRIV_RB; k++) {
					uint32_t r = rb + k * NC;
					ok[k] = r < rows_in_tile;
					row[k] = ok[k] ? r : 0;
					sl[k] = 0;
				}
#pragma unroll
				for (int j = 0; j < PRIV_DIRECT_KEYS; j++) {
					if (j < PD.nkeys) {
						const unsigned char *col = stage + R.key_smem_off[j];
						const uint8_t *lj = lut + PD.lut_off[j];
						switch (R.key_width[j]) {
						case 1:
							direct_codes<uint8_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
							break;
						case 2:
							direct_codes<uint16_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
							break;
						case 4:
							direct_codes<uint32_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
							break;
						default:
							direct_codes<uint64_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
							break;
						}
					}
				}
#pragma unroll
				for (int k = 0; k < PRIV_RB; k++) {
					slot[k] = ok[k] ? sl[k] : -1;
				}
			}
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				uint32_t r = rb + k * NC;
				live[k] = r < rows_in_tile;
				r = live[k] ? r : 0;
				unsigned long long kk = 0;
				if constexpr (KW == 1) {
#pragma unroll
					for (int j = 0; j < 4; j++) {
						if (j < R.nkeys) {
							kk |= (unsigned long long)stage[R.key_smem_off[j] + r] << (8 * j);
						}
					}
				} else if constexpr (KW == 4) {
					kk = *(const uint32_t *)(stage + R.key_smem_off[0] + (size_t)r * 4);
				} else if constexpr (KW == 2) {
					// slots were computed above; the packed key is only needed by rows that miss (below)
				} else {
#pragma unroll 1
					for (int j = 0; j < R.nkeys; j++) {
						kk |= stage_load_uint(stage + R.key_smem_off[j] + r * R.key_width[j], R.key_width[j]) << R.key_shift[j];
					}
				}
				key[k] = kk;
#pragma unroll
				for (int j = 0; j < NSUM; j++) {
					x[k][j] = *(const uint64_t *)(stage + R.sum_smem_off[j] + (size_t)r * 8);
				}
			}
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				uint64_t big = 0;
#pragma unroll
				for (int j = 0; j < NSUM; j++) {
					big |= reg_value_too_big(x[k][j], (R.sum_unsigned >> j) & 1);
				}
				if (KW != 2) {
					slot[k] = -1;
				}
				if (!live[k] || big) {
					slot[k] = -1;
				}
				if (live[k]) {
					if (!big) {
						if (KW != 2) {
							slot[k] = priv_lookup(S, slot_key, SLOTS, key[k]);
						}
						missed += slot[k] < 0 ? 1 : 0;
					}
					if (slot[k] < 0) {
						uint32_t r = rb + k * NC;
						if constexpr (KW == 2) {
							unsigned long long kk = 0;
#pragma unroll 1
							for (int j = 0; j < R.nkeys; j++) {
								kk |= stage_load_uint(stage + R.key_smem_off[j] + r * R.key_width[j], R.key_width[j]) << R.key_shift[j];
							}
							key[k] = kk;
						}
						uint64_t kw[KEY_WORDS_MAX] = {key[k], 0, 0, 0};
						row_to_global(A, stage, r, row0 + r, kw);
					}
				}
			}
			// 2. read-modify-write of the thread's private states, row after row (two rows may share a slot)
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				if (slot[k] >= 0) {
					uint64_t *a = acc + (size_t)slot[k] * NSUM * NC + tid;
#pragma unroll
					for (int j = 0; j < NSUM; j++) {
						a[(size_t)j * NC] += x[k][j];
					}
					rowc[(size_t)slot[k] * NC + tid] += 1;
				}
			}
		}
	});

	if (missed) {
		atomicAdd(&A.counters[1], missed);
	}
	__syncthreads();
	// flush: consumer warp w reduces slots w, w + nwarps, ...; lane l sums threads l, l + 32, ...
	const int lane = tid & 31, warp = tid >> 5, nwarps = NC / 32;
	if (tid < NC) {
		for (int s = warp; s < SLOTS; s += nwarps) {
			if (slot_key[s] == 0ULL) {
				continue;
			}
			unsigned long long rows = 0;
			for (int t = lane; t < NC; t += 32) {
				rows += rowc[(size_t)s * NC + t];
			}
			for (int off = 16; off; off >>= 1) {
				rows += __shfl_xor_sync(0xffffffffu, rows, off);
			}
			if (rows == 0) {
				continue;
			}
			uint64_t gkw[KEY_WORDS_MAX] = {slot_key[s] & PRIV_KEYMASK, 0, 0, 0};
			uint64_t gs = 0;
			if (lane == 0) {
				gs = agg_find_or_create(A.T, L, hash_packed_key(L, gkw), gkw, ~0ULL);
			}
			gs = __shfl_sync(0xffffffffu, gs, 0);
			uint64_t *grow = A.T.slots + gs * (uint64_t)L.stride;
			if (lane == 0) {
				atomicAdd((unsigned long long *)(grow + L.rows_off), rows);
			}
#pragma unroll
			for (int j = 0; j < NSUM; j++) {
				uint64_t lo = 0, hi = 0;
				for (int t = lane; t < NC; t += 32) {
					uint64_t v = acc[((size_t)s * NSUM + j) * NC + t];
					uint64_t nl = lo + v;
					hi += ((int64_t)v < 0 ? ~0ULL : 0ULL) + (nl < lo ? 1 : 0); // partials are signed 64-bit (reg_value_too_big)
					lo = nl;
				}
				for (int off = 16; off; off >>= 1) {
					uint64_t olo = __shfl_xor_sync(0xffffffffu, lo, off);
					uint64_t ohi = __shfl_xor_sync(0xffffffffu, hi, off);
					uint64_t nl = lo + olo;
					hi += ohi + (nl < lo ? 1 : 0);
					lo = nl;
				}
				if (lane == 0) {
					uint64_t *st = grow + L.sum_off[R.in_of_sum[j]];
					atomic_add_128(st, st + 1, lo, hi);
				}
			}
		}
	}
}

// ------------------------------------------------------------------ WPRIV: warp-private accumulators
// PRIV gives every THREAD its own copy of every slot: 35 groups x 5 sums need 1.5 KB per thread, so only 96 threads
// fit an SM and the kernel crawls.  WPRIV keeps one copy per WARP ([warp][slot][sum]: 16 warps x 36
// slots x 5 sums = 23 KB) and lets the lanes of a warp that hit the same slot take turns: ONE match.any tells every
// lane which lanes share its slot, lane `rank r` of each such set updates the state in round r with plain
// LDS / IADD / STS - in a round every active lane works on a different slot, so there is nothing to lose and nothing
// to lock.  Rounds = the largest set (3-4 for 35 uniformly spread groups).  Needs the DIRECT slot tables.
// This is the "warp-level match primitive for group matching" of BASELINE.json's north_star.
template <int NSUM>
__global__ void __launch_bounds__(512 + 32, 1)
    agg_wpriv_kernel(const __grid_constant__ TileArgs A, const __grid_constant__ RegLayout R, int SLOTS, int NC,
                     const __grid_constant__ PrivDirect PD) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * AT_MAX_STAGES];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = NC / 32;
	const AggLayout &L = A.L;
	uint64_t *acc = (uint64_t *)smem_raw;                              // [warp][slot][sum]
	uint32_t *rowc = (uint32_t *)(acc + (size_t)nwarps * SLOTS * NSUM); // [warp][slot]
	size_t state_bytes = (size_t)nwarps * SLOTS * NSUM * 8 + (size_t)nwarps * SLOTS * 4;
	uint8_t *lut = smem_raw + ((state_bytes + 15) & ~(size_t)15);
	unsigned char *stages = smem_raw + ((((state_bytes + 15) & ~(size_t)15) + PD.lut_bytes + 127) & ~(size_t)127);
	for (size_t i = tid; i < (size_t)nwarps * SLOTS * NSUM; i += blockDim.x) {
		acc[i] = 0;
	}
	for (size_t i = tid; i < (size_t)nwarps * SLOTS; i += blockDim.x) {
		rowc[i] = 0;
	}
	for (uint32_t i = tid; i < PD.lut_bytes; i += blockDim.x) {
		lut[i] = PD.lut[i];
	}
	unsigned long long missed = 0;
	__syncthreads();

	tp_tile_loop(A.tc, A.stages, stages, bars, A.row_begin, A.row_end, NC,
	             [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		// uniform trip count: match.any / reduce are warp-collectives
		for (uint32_t rb0 = 0; rb0 < rows_in_tile; rb0 += PRIV_RB * NC) {
			int slot[PRIV_RB];
			uint64_t x[PRIV_RB][NSUM];
			uint32_t row[PRIV_RB];
			int sl[PRIV_RB];
			bool ok[PRIV_RB];
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				const uint32_t r0 = rb0 + tid + k * NC;
				ok[k] = r0 < rows_in_tile;
				row[k] = ok[k] ? r0 : 0;
				sl[k] = 0;
			}
			// slot = sum of code x stride over the key columns; the width dispatch is outside the row loop
#pragma unroll
			for (int j = 0; j < PRIV_DIRECT_KEYS; j++) {
				if (j < PD.nkeys) {
					const unsigned char *col = stage + R.key_smem_off[j];
					const uint8_t *lj = lut + PD.lut_off[j];
					switch (R.key_width[j]) {
					case 1:
						direct_codes<uint8_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
						break;
					case 2:
						direct_codes<uint16_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
						break;
					case 4:
						direct_codes<uint32_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
						break;
					default:
						direct_codes<uint64_t>(col, lj, PD.kmin[j], PD.range[j], PD.stride[j], row, sl, ok);
						break;
					}
				}
			}
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				const uint32_t r0 = rb0 + tid + k * NC;
				const bool live = r0 < rows_in_tile;
				const uint32_t r = row[k];
				uint64_t big = 0;
#pragma unroll
				for (int j = 0; j < NSUM; j++) {
					x[k][j] = *(const uint64_t *)(stage + R.sum_smem_off[j] + (size_t)r * 8);
					big |= reg_value_too_big(x[k][j], (R.sum_unsigned >> j) & 1);
				}
				slot[k] = ok[k] && !big ? sl[k] : -1;
				if (live && slot[k] < 0) {
					missed += big ? 0 : 1;
					unsigned long long kk = 0; // the packed key is only needed on this (rare) path
#pragma unroll 1
					for (int j = 0; j < R.nkeys; j++) {
						kk |= stage_load_uint(stage + R.key_smem_off[j] + r * R.key_width[j], R.key_width[j]) << R.key_shift[j];
					}
					uint64_t kw[KEY_WORDS_MAX] = {kk, 0, 0, 0};
					row_to_global(A, stage, r, row0 + r, kw);
				}
			}
#pragma unroll
			for (int k = 0; k < PRIV_RB; k++) {
				const int sl = slot[k];
				const uint32_t peers = __match_any_sync(0xffffffffu, sl);
				const uint32_t rank = __popc(peers & ((1u << lane) - 1));
				const uint32_t rounds = __reduce_max_sync(0xffffffffu, sl >= 0 ? (uint32_t)__popc(peers) : 0u);
				uint64_t *a = acc + ((size_t)warp * SLOTS + (sl < 0 ? 0 : sl)) * NSUM;
				uint32_t *rc = rowc + (size_t)warp * SLOTS + (sl < 0 ? 0 : sl);
				for (uint32_t rd = 0; rd < rounds; rd++) {
					if (sl >= 0 && rank == rd) {
#pragma unroll
						for (int j = 0; j < NSUM; j++) {
							a[j] += x[k][j];
						}
						*rc += 1;
					}
					__syncwarp();
				}
			}
		}
	});

	if (missed) {
		atomicAdd(&A.counters[1], missed);
	}
	__syncthreads();
	// flush: consumer warp w reduces slots w, w + nwarps, ...; lane l < nwarps holds warp l's copy
	if (tid < NC) {
		for (int s = warp; s < SLOTS; s += nwarps) {
			unsigned long long key = PD.slot_keys[s];
			unsigned long long rows = lane < nwarps ? rowc[(size_t)lane * SLOTS + s] : 0;
			for (int off = 16; off; off >>= 1) {
				rows += __shfl_xor_sync(0xffffffffu, rows, off);
			}
			if (rows == 0 || key == 0ULL) {
				continue;
			}
			uint64_t gkw[KEY_WORDS_MAX] = {key & PRIV_KEYMASK, 0, 0, 0};
			uint64_t gs = 0;
			if (lane == 0) {
				gs = agg_find_or_create(A.T, L, hash_packed_key(L, gkw), gkw, ~0ULL);
			}
			gs = __shfl_sync(0xffffffffu, gs, 0);
			uint64_t *grow = A.T.slots + gs * (uint64_t)L.stride;
			if (lane == 0) {
				atomicAdd((unsigned long long *)(grow + L.rows_off), rows);
			}
#pragma unroll
			for (int j = 0; j < NSUM; j++) {
				uint64_t lo = lane < nwarps ? acc[((size_t)lane * SLOTS + s) * NSUM + j] : 0;
				uint64_t hi = (int64_t)lo < 0 ? ~0ULL : 0ULL; // partials are signed 64-bit values (reg_value_too_big)
				for (int off = 16; off; off >>= 1) {
					uint64_t olo = __shfl_xor_sync(0xffffffffu, lo, off);
					uint64_t ohi = __shfl_xor_sync(0xffffffffu, hi, off);
					uint64_t nl = lo + olo;
					hi += ohi + (nl < lo ? 1 : 0);
					lo = nl;
				}
				if (lane == 0) {
					uint64_t *st = grow + L.sum_off[R.in_of_sum[j]];
					atomic_add_128(st, st + 1, lo, hi);
				}
			}
		}
	}
}

template <int NSUM>
static int launch_wpriv(b200_ctx *ctx, const TileArgs &A, const RegLayout &R, int slots, int nc, size_t smem, unsigned grid,
                        const PrivDirect &PD) {
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(agg_wpriv_kernel<NSUM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
		attr_set = true;
	}
	agg_wpriv_kernel<NSUM><<<grid, nc + 32, smem, ctx->stream>>>(A, R, slots, nc, PD);
	return B200_OK;
}

// dynamic shared memory available to the kernel: 227 KB per CTA minus its static part (directory, barriers)
#define PRIV_DYN_SMEM (227 * 1024 - (int)sizeof(PrivShared) - 1024)

// Largest configuration that fits: returns consumer threads (0 = does not fit) for `slots` private slots.
static int priv_pick_threads(int nsum, int slots, uint32_t row_bytes, uint32_t *tile_rows, int *stages, size_t extra = 0) {
	const int cand[] = {512, 384, 256, 192, 128, 96, 64};
	for (int nc : cand) {
		size_t state = (size_t)slots * nsum * nc * 8 + (size_t)slots * nc * 4 + (size_t)slots * 8 + 128 + extra;
		for (uint32_t rpt = 4; rpt >= 2; rpt -= 2) {
			uint32_t rows = (uint32_t)nc * rpt;
			if (rows % 128) {
				rows = (rows + 127) / 128 * 128; // the ragged part of a thread's PRIV_RB rows is masked off in the kernel
			}
			for (int st = 3; st >= 2; st--) {
				size_t need = state + (size_t)st * (((size_t)rows * row_bytes + 16 * TP_MAX_COLS + 127) & ~(size_t)127) + 512;
				if (need <= PRIV_DYN_SMEM) {
					*tile_rows = rows;
					*stages = st;
					return nc;
				}
			}
		}
	}
	return 0;
}

// how many groups the PRIV path can keep per CTA for this layout (0 = not eligible); used by b200_agg_sink's adaptation
int b200_agg_priv_capacity(const AggLayout &L) {
	int nsum = 0;
	uint32_t row_bytes = 0;
	if (L.key_bytes > 7) {
		return 0;
	}
	for (int j = 0; j < L.nkeys; j++) {
		if (!b200_type_is_integer(L.key_type[j])) {
			return 0;
		}
		row_bytes += b200_type_size(L.key_type[j]);
	}
	for (int i = 0; i < L.ninputs; i++) {
		if (!b200_type_is_integer(L.input_type[i]) || L.min_off[i] >= 0 || L.max_off[i] >= 0) {
			return 0;
		}
		if (L.sum_off[i] >= 0) {
			if (b200_type_size(L.input_type[i]) != 8) {
				return 0;
			}
			nsum++;
		}
		row_bytes += b200_type_size(L.input_type[i]);
	}
	if (nsum < 1 || nsum > REG_MAX_SUMS) {
		return 0;
	}
	int best = 0;
	for (int slots = 8; slots <= 128; slots += 4) {
		uint32_t tr;
		int st;
		if (priv_pick_threads(nsum, slots, row_bytes, &tr, &st) >= 64) {
			best = slots;
		}
	}
	// warp-private copies (WPRIV, needs the direct slot tables): 8 warps x slots x (8 nsum + 4) bytes next to the stages
	int wslots = (int)((176 * 1024) / (8 * (nsum * 8 + 4)));
	wslots = wslots > 1024 ? 1024 : wslots;
	best = best > wslots ? best : wslots;
	return best;
}

template <int NSUM, int KW>
static int launch_priv(b200_ctx *ctx, const TileArgs &A, const RegLayout &R, int slots, int nc, size_t smem, unsigned grid,
                       const PrivDirect &PD) {
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(agg_priv_kernel<NSUM, KW>, cudaFuncAttributeMaxDynamicSharedMemorySize, PRIV_DYN_SMEM));
		attr_set = true;
	}
	agg_priv_kernel<NSUM, KW><<<grid, nc + 32, smem, ctx->stream>>>(A, R, slots, nc, PD);
	return B200_OK;
}

template <int KW>
static int dispatch_priv(b200_ctx *ctx, const TileArgs &A, const RegLayout &R, int slots, int nc, size_t smem, unsigned grid,
                         const PrivDirect &PD) {
	switch (R.nsum) {
	case 1:
		return launch_priv<1, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	case 2:
		return launch_priv<2, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	case 3:
		return launch_priv<3, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	case 4:
		return launch_priv<4, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	case 5:
		return launch_priv<5, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	default:
		return launch_priv<6, KW>(ctx, A, R, slots, nc, smem, grid, PD);
	}
}

// Called by b200_agg_tile_sink (mode 2).  A arrives with keys / inputs registered as tile columns (A.tc, A.sm).
// Returns B200_ERR_INVALID when the shape is not eligible (the caller falls back to MID).
int b200_agg_priv_launch(b200_ctx *ctx, TileArgs &A, const AggLayout &L, const KeyCols &keys, const AggCols &ac, int groups_hint,
                         const PrivDirect *direct) {
	RegLayout R;
	memset(&R, 0, sizeof(R));
	if (L.key_bytes > 7) {
		return B200_ERR_INVALID;
	}
	R.nkeys = L.nkeys;
	for (int j = 0; j < L.nkeys; j++) {
		if (!b200_type_is_integer(L.key_type[j]) || keys.c[j].validity) {
			return B200_ERR_INVALID;
		}
		R.key_width[j] = b200_type_size(L.key_type[j]);
		R.key_shift[j] = L.key_off[j] * 8;
	}
	for (int i = 0; i < L.ninputs; i++) {
		if (!b200_type_is_integer(L.input_type[i]) || ac.track_cnt[i] || ac.c[i].validity || L.min_off[i] >= 0 ||
		    L.max_off[i] >= 0) {
			return B200_ERR_INVALID;
		}
		if (L.sum_off[i] >= 0) {
			if (R.nsum >= REG_MAX_SUMS || b200_type_size(L.input_type[i]) != 8) {
				return B200_ERR_INVALID;
			}
			R.sum_unsigned |= (b200_type_is_unsigned_int(L.input_type[i]) ? 1u : 0u) << R.nsum;
			R.in_of_sum[R.nsum++] = i;
		}
	}
	if (R.nsum < 1) {
		return B200_ERR_INVALID;
	}
	uint32_t row_bytes = 0;
	for (int i = 0; i < A.tc.n; i++) {
		row_bytes += A.tc.c[i].width;
	}
	// slots: the group count seen by the adaptation probe, with some slack for groups that show up later
	int cap = b200_agg_priv_capacity(L);
	int slots = groups_hint + 2; // a little slack for groups that only show up after the adaptation probe
	slots = (slots + 1) & ~1;
	PrivDirect PD;
	memset(&PD, 0, sizeof(PD));
	if (direct && direct->nslots > 0 && !getenv("B200_AGG_NO_DIRECT")) {
		PD = *direct;
		slots = (PD.nslots + 1) & ~1;
	}
	if (slots > cap) {
		slots = cap;
	}
	if (slots < 8) {
		slots = 8;
	}
	// thread-private copies when >= 256 threads' worth of them fit (no bank conflicts, no rounds); otherwise the
	// warp-private variant
	bool thread_private_fits = false;
	if (PD.nslots) {
		uint32_t tr0 = 0;
		int st0 = 0;
		thread_private_fits = priv_pick_threads(R.nsum, slots, row_bytes, &tr0, &st0, PD.lut_bytes + 16) >= 256;
	}
	const char *wenv = getenv("B200_AGG_WPRIV"); // 1 = always, 0 = never (same as B200_AGG_NO_WPRIV)
	bool use_wpriv = PD.nslots && !getenv("B200_AGG_NO_WPRIV") && !(wenv && atoi(wenv) == 0) &&
	                 (!thread_private_fits || (wenv && atoi(wenv) == 1));
	if (use_wpriv) {
		// warp-private accumulators: 16 warps unless the states of that many copies do not fit
		for (int wnc = 512; wnc >= 128; wnc -= 128) {
			size_t st = (size_t)(wnc / 32) * slots * (R.nsum * 8 + 4);
			st = ((st + 15) & ~(size_t)15) + PD.lut_bytes;
			uint32_t rows = (uint32_t)wnc * 4;
			tile_cols_finish(&A.tc, rows);
			for (int sg = 3; sg >= 2; sg--) {
				size_t smem_w = ((st + 127) & ~(size_t)127) + (size_t)sg * A.tc.stage_bytes;
				if (smem_w > 216 * 1024) {
					continue;
				}
				A.stages = sg;
				for (int j = 0; j < L.nkeys; j++) {
					R.key_smem_off[j] = A.tc.c[A.sm.key_data[j]].smem_off;
				}
				for (int j = 0; j < R.nsum; j++) {
					R.sum_smem_off[j] = A.tc.c[A.sm.in_data[R.in_of_sum[j]]].smem_off;
				}
				uint64_t nrows = A.row_end - A.row_begin;
				uint64_t nt = (nrows + rows - 1) / rows;
				unsigned g = (unsigned)(nt < (uint64_t)ctx->sm_count ? nt : (uint64_t)ctx->sm_count);
				int rcw;
				switch (R.nsum) {
				case 1:
					rcw = launch_wpriv<1>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				case 2:
					rcw = launch_wpriv<2>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				case 3:
					rcw = launch_wpriv<3>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				case 4:
					rcw = launch_wpriv<4>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				case 5:
					rcw = launch_wpriv<5>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				default:
					rcw = launch_wpriv<6>(ctx, A, R, slots, wnc, smem_w, g, PD);
					break;
				}
				B200_TRY(rcw);
				CUDA_TRY(cudaGetLastError());
				return B200_OK;
			}
		}
	}
	uint32_t tile_rows = 0;
	int stages = 0;
	int nc = priv_pick_threads(R.nsum, slots, row_bytes, &tile_rows, &stages, PD.nslots ? PD.lut_bytes + 16 : 0);
	if (nc < 64) {
		return B200_ERR_INVALID;
	}
	tile_cols_finish(&A.tc, tile_rows);
	A.stages = stages;
	for (int j = 0; j < L.nkeys; j++) {
		R.key_smem_off[j] = A.tc.c[A.sm.key_data[j]].smem_off;
	}
	for (int j = 0; j < R.nsum; j++) {
		R.sum_smem_off[j] = A.tc.c[A.sm.in_data[R.in_of_sum[j]]].smem_off;
	}
	size_t state = (size_t)slots * R.nsum * nc * 8 + (size_t)slots * nc * 4 + (size_t)slots * 8;
	if (PD.nslots) {
		state = ((state + 15) & ~(size_t)15) + PD.lut_bytes;
	}
	size_t smem = ((state + 127) & ~(size_t)127) + (size_t)stages * A.tc.stage_bytes;
	if (smem > (size_t)PRIV_DYN_SMEM) {
		return B200_ERR_INVALID;
	}
	uint64_t n = A.row_end - A.row_begin;
	uint64_t ntiles = (n + tile_rows - 1) / tile_rows;
	unsigned grid = (unsigned)(ntiles < (uint64_t)ctx->sm_count ? ntiles : (uint64_t)ctx->sm_count);
	bool all1 = R.nkeys <= 4;
	for (int j = 0; j < R.nkeys; j++) {
		all1 = all1 && R.key_width[j] == 1 && R.key_shift[j] == (uint32_t)(8 * j);
	}
	int rc;
	if (PD.nslots) {
		rc = dispatch_priv<2>(ctx, A, R, slots, nc, smem, grid, PD);
	} else if (all1) {
		rc = dispatch_priv<1>(ctx, A, R, slots, nc, smem, grid, PD);
	} else if (R.nkeys == 1 && R.key_width[0] == 4 && R.key_shift[0] == 0) {
		rc = dispatch_priv<4>(ctx, A, R, slots, nc, smem, grid, PD);
	} else {
		rc = dispatch_priv<0>(ctx, A, R, slots, nc, smem, grid, PD);
	}
	B200_TRY(rc);
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// Build the DIRECT addressing tables from the packed keys (kw0) of the groups discovered so far.  Returns false when
// the shape does not qualify (a key column spreads over more than PRIV_LUT_MAX values, more than 4 key columns, the
// code space exceeds `max_slots`).  out_tables receives lut bytes followed (8-byte aligned) by the slot keys; the
// caller uploads it and patches PD->lut / PD->slot_keys.
bool b200_agg_priv_build_direct(const AggLayout &L, const uint64_t *kw0, int ngroups, int max_slots, PrivDirect *PD,
                                std::vector<uint8_t> *out_tables) {
	memset(PD, 0, sizeof(*PD));
	if (L.nkeys > PRIV_DIRECT_KEYS || L.key_bytes > 7 || ngroups < 1) {
		return false;
	}
	std::vector<std::vector<uint64_t>> vals(L.nkeys);
	for (int j = 0; j < L.nkeys; j++) {
		int sz = b200_type_size(L.key_type[j]);
		uint64_t m = sz >= 8 ? ~0ULL : ((1ULL << (sz * 8)) - 1);
		for (int g = 0; g < ngroups; g++) {
			vals[j].push_back((kw0[g] >> (L.key_off[j] * 8)) & m);
		}
	}
	uint32_t lut_total = 0;
	std::vector<std::vector<uint64_t>> distinct(L.nkeys);
	long long nslots = 1;
	for (int j = L.nkeys - 1; j >= 0; j--) {
		std::vector<uint64_t> d = vals[j];
		std::sort(d.begin(), d.end());
		d.erase(std::unique(d.begin(), d.end()), d.end());
		uint64_t range = d.back() - d.front() + 1;
		if (range > PRIV_LUT_MAX || d.size() > 254) {
			return false;
		}
		PD->kmin[j] = d.front();
		PD->range[j] = (uint32_t)range;
		PD->stride[j] = (uint32_t)nslots;
		nslots *= (long long)d.size();
		if (nslots > max_slots) {
			return false;
		}
		distinct[j] = d;
	}
	for (int j = 0; j < L.nkeys; j++) {
		PD->lut_off[j] = lut_total;
		lut_total += PD->range[j];
	}
	PD->nkeys = L.nkeys;
	PD->nslots = (int)nslots;
	PD->lut_bytes = (lut_total + 7) & ~7u;
	out_tables->assign(PD->lut_bytes + (size_t)(((int)nslots + 1) & ~1) * 8, 0xff);
	for (int j = 0; j < L.nkeys; j++) {
		for (size_t c = 0; c < distinct[j].size(); c++) {
			(*out_tables)[PD->lut_off[j] + (distinct[j][c] - PD->kmin[j])] = (uint8_t)c;
		}
	}
	// slot keys: every code combination is a potential group (its key is well defined even if no row has shown it yet)
	unsigned long long *sk = (unsigned long long *)(out_tables->data() + PD->lut_bytes);
	for (long long s = 0; s < ((nslots + 1) & ~1LL); s++) {
		unsigned long long key = 0;
		if (s < nslots) {
			for (int j = 0; j < L.nkeys; j++) {
				size_t c = (size_t)((s / PD->stride[j]) % (long long)distinct[j].size());
				key |= distinct[j][c] << (L.key_off[j] * 8);
			}
			key |= 1ULL << 56;
		}
		sk[s] = key;
	}
	return true;
}
