// K6 sink path HC: high-cardinality groups (TPC-H Q3: millions of groups) in an L2-FIRST structure-of-arrays table.
//
// What a random table access costs is the NUMBER of L2 transactions per row and whether the touched footprint stays
// inside L2 (50 MB on an H100) - not sector locality; scripts/ubench/atomics.cu measures both against the table size
// (not yet run on H100).  The generic table of agg.cu (one 64-128 byte row per group holding tag, key, hash,
// rows, cnt and 128-bit sums updated with value-returning atomics) costs ~6 transactions per row and outgrows L2 at
// 1 M groups.  This path therefore keeps, per group, only what the row path touches, each in its own dense array:
//   keys[cap][KW]  the packed group key (1 or 2 words); bits 6/7 of its NULL-flag byte are OCCUPIED / LOCKED, so the
//                  key block is its own tag: a probe is ONE 8- or 16-byte load
//   A[i][cap]      per summed input: sum of the values' LOW 32 bits   (one RED, no carry, no return value)
//   B[i][cap]      per summed input: sum of the values' HIGH 32 bits  (RED only when that half is non-zero: DECIMAL /
//                  BIGINT measures below 2^32 never touch it)          sum = A + (B << 32) in 128 bits
//   rows[cap]      only when an aggregate needs a count (COUNT / COUNT(*) / AVG); cnt[i][cap] only for nullable inputs
// TPC-H Q3's group-by (keys i64 + u16 + u8, one SUM): 16 B load + 1 RED per row; 1 M groups = 48 MB, about the size of
// an H100's 50 MB L2, so with the input streaming past it cannot all stay resident (how much does is not measured).
// The table is an accumulation front end: b200_agg_finalize / export / combine first merge it into the generic table
// (agg_hc_flush_kernel), so everything downstream of the sink is unchanged.  Rows that find the table at its fill
// limit are DEFERRED (their row ids are appended to a list, one atomic per warp); the host doubles the table (rehash)
// and replays them (agg_hc_rows_kernel), like the generic path's growth protocol.  The group counter is sharded 64
// ways (one shard per CTA residue) so that inserts do not serialise on one L2 address.
// Reference semantics: GroupedAggregateHashTable::FindOrCreateGroupsInternal / UpdateAggregates
// (src/execution/aggregate_hashtable.cpp:803-977,688-722), hugeint sums (sum_helpers.hpp:155-215); the reference's
// own answer to tables that outgrow the cache is radix partitioning (radix_partitioned_hashtable.cpp:790-876).
#include "agg_tile.cuh"
#include <cstring>
#include <cstdlib>

#define HC_THREADS 256
#define HC_RB 4
#define HC_MIN_CAP (1ULL << 20) // zeroing 1 M slots costs ~20 us; saves four doublings on every high-cardinality input
#define HC_SHARDS 64 // group-count shards, 32 bytes apart

struct HcView {
	uint64_t *keys;
	uint64_t *rows;
	uint64_t *A[MAX_INPUTS];
	uint64_t *B[MAX_INPUTS];
	uint64_t *cnt[MAX_INPUTS];
	uint64_t mask;
	unsigned long long *count; // HC_SHARDS counters, 4 words apart
	uint64_t limit;            // groups per shard
	uint64_t occ_bit, lock_bit; // inside the last key word
};

struct AggHc {
	void *pinned_mem; // table memory currently covered by the stream's persisting-L2 window (nullptr: none)
	size_t hot_bytes; // keys + rows + low halves + counts: what the row path touches
	HcView V;
	int kw;
	uint64_t cap;
	void *mem;
	bool need_rows;
	bool track_cnt[MAX_INPUTS];
	uint64_t rows_sunk;
};

// key block stride in words: 3-word keys (e.g. Q3's BIGINT + DATE + INTEGER before type compression) use 32-byte blocks
#define HC_KWS(KW) ((KW) == 3 ? 4 : (KW))

// ONE slot hash for every kernel that touches the table (sink, replay, rehash): multiply-xorshift-multiply of the key
// words.  (The tight kernel briefly used its own function: keys re-inserted after a rehash were not found, the table
// filled up with duplicates - still merged correctly by the flush, but 2x slower.)
__device__ __forceinline__ uint64_t hc_hash_words(uint64_t k0, uint64_t k1, uint64_t k2, int KW) {
	uint64_t x = k0;
	if (KW >= 2) {
		x ^= k1 * 0x9e3779b97f4a7c15ULL;
	}
	if (KW >= 3) {
		x ^= k2 * 0xc2b2ae3d27d4eb4fULL;
	}
	x *= 0xd6e8feb86659fd93ULL;
	x ^= x >> 32;
	x *= 0xd6e8feb86659fd93ULL;
	return x ^ (x >> 29);
}

__device__ __forceinline__ uint64_t hc_hash(const uint64_t kw[KEY_WORDS_MAX], int KW) {
	return hc_hash_words(kw[0], kw[1], kw[2], KW);
}

// w[] receives the slot's key words (one or two 16-byte loads, or one 8-byte load)
template <int KW>
__device__ __forceinline__ void hc_load_keys(const HcView &H, uint64_t slot, uint64_t (&w)[3]) {
	const uint64_t *p = H.keys + slot * HC_KWS(KW);
	if (KW == 1) {
		asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(w[0]) : "l"(p) : "memory");
	} else {
		asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(w[0]), "=l"(w[1]) : "l"(p) : "memory");
		if (KW == 3) {
			uint64_t spare;
			asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(w[2]), "=l"(spare) : "l"(p + 2) : "memory");
		}
	}
}

// Slot of the group with packed key kw (starting at `slot`, whose key words were already loaded into w[]),
// inserting it if needed; SLOT_DEFER when the table is at its fill limit.
template <int KW>
__device__ __forceinline__ uint64_t hc_find_or_create(const HcView &H, const uint64_t kw[KEY_WORDS_MAX], uint64_t slot,
                                                      uint64_t (&w)[3]) {
	const uint64_t mine = kw[KW - 1] | H.occ_bit;
	unsigned long long *const shard = H.count + (blockIdx.x % HC_SHARDS) * 4;
	while (true) {
		uint64_t last = w[KW - 1];
		unsigned long long *p = (unsigned long long *)(H.keys + slot * HC_KWS(KW));
		if (last == 0) {
			// reserve a group BEFORE claiming the slot, so that the fill limit is exact (a full table would never
			// terminate the probe loop)
			if (*(volatile unsigned long long *)shard >= H.limit) {
				return SLOT_DEFER;
			}
			unsigned long long c = atomicAdd(shard, 1ULL);
			if (c >= H.limit) {
				atomicAdd(shard, ~0ULL);
				return SLOT_DEFER;
			}
			unsigned long long old = atomicCAS(&p[KW - 1], 0ULL, (unsigned long long)(mine | H.lock_bit));
			if (old == 0ULL) {
				if (KW >= 2) {
#pragma unroll
					for (int q = 0; q < KW - 1; q++) {
						*(volatile unsigned long long *)&p[q] = kw[q];
					}
					__threadfence();
				}
				*(volatile unsigned long long *)&p[KW - 1] = mine;
				return slot;
			}
			// somebody else claimed the slot between our load and the CAS: give the reservation back and look at the
			// slot again with FRESH words (comparing the other key words from the earlier, empty read made a thread
			// walk past its own key and insert it a second time further down the probe sequence)
			atomicAdd(shard, ~0ULL);
			hc_load_keys<KW>(H, slot, w);
			continue;
		}
		if ((last & ~H.lock_bit) == mine) {
			if (KW == 1) {
				return slot; // the key is the whole block: nothing else to wait for (state arrays start zeroed)
			}
			// Hit path (every row after the first of its group): the block's words came from ONE aligned 16-byte load
			// of a published slot - no fence (a membar per row would be the hottest stall).  Only a slot seen
			// while its inserter still holds the lock waits, fences and re-reads.
			bool eq = !(last & H.lock_bit);
#pragma unroll
			for (int q = 0; q < KW - 1; q++) {
				eq = eq && w[q] == kw[q];
			}
			if (eq) {
				return slot;
			}
			if (last & H.lock_bit) {
				while (last & H.lock_bit) {
					last = *(volatile unsigned long long *)&p[KW - 1];
				}
				__threadfence();
				eq = true;
#pragma unroll
				for (int q = 0; q < KW - 1; q++) {
					eq = eq && *(volatile unsigned long long *)&p[q] == kw[q];
				}
				if (eq) {
					return slot;
				}
			}
		}
		slot = (slot + 1) & H.mask;
		hc_load_keys<KW>(H, slot, w);
	}
}

// a + (b << 32) in 128 bits (b is a signed sum of high halves for signed inputs)
__device__ __forceinline__ void hc_sum128(int type, uint64_t a, uint64_t b, uint64_t *lo, uint64_t *hi) {
	uint64_t blo = b << 32;
	uint64_t bhi = b200_type_is_signed_int(type) ? (uint64_t)((int64_t)b >> 32) : (b >> 32);
	*lo = a + blo;
	*hi = bhi + (*lo < a ? 1 : 0);
}

// fire-and-forget state updates of one row (slot s): REDs only
__device__ __forceinline__ void hc_apply(const HcView &H, const AggLayout &L, uint64_t s, int i, uint64_t raw) {
	if (H.cnt[i]) {
		atomicAdd((unsigned long long *)(H.cnt[i] + s), 1ULL);
	}
	if (H.A[i]) {
		atomicAdd((unsigned long long *)(H.A[i] + s), (unsigned long long)(raw & 0xffffffffULL));
		uint64_t hi = b200_type_is_signed_int(L.input_type[i]) ? (uint64_t)((int64_t)raw >> 32) : (raw >> 32);
		if (hi) {
			atomicAdd((unsigned long long *)(H.B[i] + s), (unsigned long long)hi);
		}
	}
}

// append the deferred rows of a warp to the list with ONE atomic (all 32 lanes must call this together)
__device__ __forceinline__ void hc_defer_rows(uint32_t *deferred, unsigned long long *counter, const uint32_t *rows, int n) {
	const int lane = threadIdx.x & 31;
	uint32_t incl = (uint32_t)n;
#pragma unroll
	for (int off = 1; off < 32; off <<= 1) {
		uint32_t v = __shfl_up_sync(0xffffffffu, incl, off);
		if (lane >= off) {
			incl += v;
		}
	}
	uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
	if (total == 0) {
		return;
	}
	unsigned long long base = 0;
	if (lane == 0) {
		base = atomicAdd(counter, (unsigned long long)total);
	}
	base = __shfl_sync(0xffffffffu, base, 0) + incl - n;
	for (int k = 0; k < n; k++) {
		deferred[base + k] = rows[k];
	}
}

// One probe step of row state (slot, w[]): -1 = keep probing (slot advanced, next key block loaded), else the slot or
// SLOT_DEFER.  The body of hc_find_or_create's loop, split out so that a thread can advance ALL its rows one step per
// round: the rows' dependent L2 loads overlap, and a warp's trip count is the longest probe sequence of any of its
// rows instead of the sum over the rows of the per-row maxima (per-lane probe loops leave most lanes idle).
#define HC_PENDING 0xfffffffffffffffeULL
template <int KW>
__device__ __forceinline__ uint64_t hc_probe_step(const HcView &H, const uint64_t kw[KEY_WORDS_MAX], uint64_t &slot,
                                                  uint64_t (&w)[3]) {
	const uint64_t mine = kw[KW - 1] | H.occ_bit;
	uint64_t last = w[KW - 1];
	if (last == 0 || (last & H.lock_bit)) {
		return hc_find_or_create<KW>(H, kw, slot, w); // rare: insert, or a slot seen mid-insert
	}
	bool eq = last == mine;
#pragma unroll
	for (int q = 0; q < KW - 1; q++) {
		eq = eq && w[q] == kw[q];
	}
	if (eq) {
		return slot;
	}
	slot = (slot + 1) & H.mask;
	hc_load_keys<KW>(H, slot, w);
	return HC_PENDING;
}

// key column descriptors of the SIMPLE path: integer keys without NULLs, packed with branch-free loads
struct HcKeyDesc {
	uint32_t smem_off[MAX_KEYS];
	uint32_t width[MAX_KEYS];
	uint32_t shift[MAX_KEYS]; // bit position inside its key word
	uint32_t word[MAX_KEYS];
	uint32_t in_off[MAX_INPUTS]; // SIMPLE inputs: 8-byte integers without NULLs
	int nkeys, ninputs;
};

// SIMPLE: integer keys without NULLs and 8-byte integer inputs without NULLs (the TPC-H / SSB shape): keys are packed
// from descriptors with branch-free loads, values are plain 64-bit loads - no per-row type dispatch.
template <int KW, bool SIMPLE>
__global__ void __launch_bounds__(HC_THREADS + 32, 2)
    agg_hc_kernel(const __grid_constant__ TileArgs A, const __grid_constant__ HcView H, const __grid_constant__ HcKeyDesc D) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * AT_MAX_STAGES];
	const int tid = threadIdx.x;
	const AggLayout &L = A.L;
	tp_tile_loop(A.tc, A.stages, smem_raw, bars, A.row_begin, A.row_end, HC_THREADS,
	             [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		// uniform trip count per warp (the deferral append is a warp-collective)
		for (uint32_t rb0 = 0; rb0 < rows_in_tile; rb0 += HC_RB * HC_THREADS) {
			const uint32_t rb = rb0 + tid;
			uint64_t kw[HC_RB][KEY_WORDS_MAX];
			uint64_t slot[HC_RB], w[HC_RB][3], found[HC_RB];
			// 1. pack the keys and issue the first key-block load of every row (HC_RB random L2 accesses in flight)
#pragma unroll
			for (int k = 0; k < HC_RB; k++) {
				uint32_t r = rb + k * HC_THREADS;
				found[k] = SLOT_DEFER - 2; // dead row
				if (r < rows_in_tile) {
					if (SIMPLE) {
						uint64_t k0 = 0, k1 = 0, k2 = 0;
#pragma unroll 1
						for (int j = 0; j < D.nkeys; j++) {
							uint64_t v = stage_load_uint(stage + D.smem_off[j] + r * D.width[j], D.width[j]) << D.shift[j];
							k0 |= D.word[j] == 0 ? v : 0;
							k1 |= D.word[j] == 1 ? v : 0;
							k2 |= D.word[j] == 2 ? v : 0;
						}
						kw[k][0] = k0;
						kw[k][1] = k1;
						kw[k][2] = k2;
						kw[k][3] = 0;
					} else {
						stage_pack_key(A, stage, r, kw[k]);
					}
					slot[k] = hc_hash(kw[k], KW) & H.mask;
					hc_load_keys<KW>(H, slot[k], w[k]);
					found[k] = HC_PENDING;
				}
			}
			// 2. resolve all rows round by round
			bool any = true;
			while (any) {
				any = false;
#pragma unroll
				for (int k = 0; k < HC_RB; k++) {
					if (found[k] == HC_PENDING) {
						found[k] = hc_probe_step<KW>(H, kw[k], slot[k], w[k]);
						any = any || found[k] == HC_PENDING;
					}
				}
			}
			// 3. fire-and-forget REDs on the state arrays; rows that found the table full are deferred
			uint32_t drows[HC_RB];
			int ndef = 0;
#pragma unroll
			for (int k = 0; k < HC_RB; k++) {
				uint32_t r = rb + k * HC_THREADS;
				uint64_t s = found[k];
				if (s == SLOT_DEFER) {
					drows[ndef++] = (uint32_t)(row0 + r);
				} else if (s != SLOT_DEFER - 2) {
					if (H.rows) {
						atomicAdd((unsigned long long *)(H.rows + s), 1ULL);
					}
					if (SIMPLE) {
#pragma unroll 1
						for (int i = 0; i < D.ninputs; i++) {
							uint64_t raw = *(const uint64_t *)(stage + D.in_off[i] + (size_t)r * 8);
							if (H.A[i]) {
								atomicAdd((unsigned long long *)(H.A[i] + s), (unsigned long long)(raw & 0xffffffffULL));
								// SIMPLE inputs are INT64 or UINT64: the high half is taken as stored (signedness is applied
								// when the halves are recombined in the flush)
								uint64_t hi = L.input_type[i] == B200_INT64 ? (uint64_t)((int64_t)raw >> 32) : (raw >> 32);
								if (hi) {
									atomicAdd((unsigned long long *)(H.B[i] + s), (unsigned long long)hi);
								}
							}
						}
					} else {
#pragma unroll 1
						for (int i = 0; i < L.ninputs; i++) {
							if (stage_valid(stage, A.tc, A.sm.in_valid[i], r)) {
								hc_apply(H, L, s, i, stage_value(stage, A.tc.c[A.sm.in_data[i]], L.input_type[i], r));
							}
						}
					}
				}
			}
			__syncwarp();
			hc_defer_rows(A.deferred, &A.counters[0], drows, ndef);
		}
	});
}

// ------------------------------------------------------------------ SIMPLE shape, tight kernel
// Integer keys without NULLs (<= 4 key columns) and <= 4 INT64 / UINT64 inputs without NULLs: the TPC-H / SSB shape.
// Same table protocol as agg_hc_kernel, but the hot loop holds nothing but the hit path: keys are packed from four
// predicated descriptor slots, the slot hash is one multiply-xorshift-multiply, inserts / locked slots / full tables go
// through ONE out-of-line call (hc_slow_path), the deferral list is built from a bit mask.  The generic kernel is issue-bound; this
// one keeps the instructions per row several times lower.
struct HcSimple {
	TileCols tc;
	int stages;
	int nkeys, ninputs;
	uint32_t key_off[4], key_width[4], key_shift[4], key_word[4];
	uint32_t in_off[4];
	uint32_t in_signed; // bit i: input i is INT64 (arithmetic high half), else UINT64
	uint64_t row_begin, row_end;
	uint32_t *deferred;
	unsigned long long *counters;
};

template <int KW>
__device__ __noinline__ uint64_t hc_slow_path(const HcView &H, uint64_t kw0, uint64_t kw1, uint64_t kw2, uint64_t slot,
                                             uint64_t w0, uint64_t w1, uint64_t w2) {
	uint64_t kw[KEY_WORDS_MAX] = {kw0, kw1, kw2, 0};
	uint64_t w[3] = {w0, w1, w2};
	return hc_find_or_create<KW>(H, kw, slot, w);
}

template <int KW>
__global__ void __launch_bounds__(HC_THREADS + 32, 2)
    agg_hc_simple_kernel(const __grid_constant__ HcSimple P, const __grid_constant__ HcView H) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * AT_MAX_STAGES];
	const int tid = threadIdx.x, lane = tid & 31;
	const uint64_t occ = H.occ_bit;
	tp_tile_loop(P.tc, P.stages, smem_raw, bars, P.row_begin, P.row_end, HC_THREADS,
	             [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		for (uint32_t rb0 = 0; rb0 < rows_in_tile; rb0 += HC_RB * HC_THREADS) {
			uint64_t k0[HC_RB], k1[HC_RB], k2[HC_RB], slot[HC_RB], w0[HC_RB], w1[HC_RB], w2[HC_RB];
			uint32_t pend = 0, live = 0, defer = 0;
#pragma unroll
			for (int k = 0; k < HC_RB; k++) {
				const uint32_t r = rb0 + tid + k * HC_THREADS;
				k0[k] = k1[k] = k2[k] = 0;
				w0[k] = w1[k] = w2[k] = 0;
				slot[k] = 0;
				if (r < rows_in_tile) {
#pragma unroll
					for (int j = 0; j < 4; j++) {
						if (j < P.nkeys) {
							uint64_t v = stage_load_uint(stage + P.key_off[j] + r * P.key_width[j], P.key_width[j]) << P.key_shift[j];
							uint32_t wd = P.key_word[j];
							k0[k] |= wd == 0 ? v : 0;
							if (KW >= 2) {
								k1[k] |= wd == 1 ? v : 0;
							}
							if (KW >= 3) {
								k2[k] |= wd == 2 ? v : 0;
							}
						}
					}
					slot[k] = hc_hash_words(k0[k], k1[k], k2[k], KW) & H.mask;
					uint64_t w[3];
					hc_load_keys<KW>(H, slot[k], w);
					w0[k] = w[0];
					if (KW >= 2) {
						w1[k] = w[1];
					}
					if (KW >= 3) {
						w2[k] = w[2];
					}
					pend |= 1u << k;
					live |= 1u << k;
				}
			}
			// resolve round by round: every pending row advances one probe step per round
			while (pend) {
#pragma unroll
				for (int k = 0; k < HC_RB; k++) {
					if (!((pend >> k) & 1)) {
						continue;
					}
					const uint64_t klast = KW == 1 ? k0[k] : (KW == 2 ? k1[k] : k2[k]);
					const uint64_t last = KW == 1 ? w0[k] : (KW == 2 ? w1[k] : w2[k]);
					bool eq = last == (klast | occ);
					if (KW >= 2) {
						eq = eq && w0[k] == k0[k];
					}
					if (KW >= 3) {
						eq = eq && w1[k] == k1[k];
					}
					if (eq) {
						pend &= ~(1u << k);
					} else if (last == 0 || (last & H.lock_bit)) {
						uint64_t s = hc_slow_path<KW>(H, k0[k], k1[k], k2[k], slot[k], w0[k], w1[k], w2[k]);
						if (s == SLOT_DEFER) {
							defer |= 1u << k;
						} else {
							slot[k] = s;
						}
						pend &= ~(1u << k);
					} else {
						slot[k] = (slot[k] + 1) & H.mask;
						uint64_t w[3];
						hc_load_keys<KW>(H, slot[k], w);
						w0[k] = w[0];
						if (KW >= 2) {
							w1[k] = w[1];
						}
						if (KW >= 3) {
							w2[k] = w[2];
						}
					}
				}
			}
			// fire-and-forget REDs
#pragma unroll
			for (int k = 0; k < HC_RB; k++) {
				if (!((live >> k) & 1) || ((defer >> k) & 1)) {
					continue;
				}
				const uint32_t r = rb0 + tid + k * HC_THREADS;
				const uint64_t s = slot[k];
				if (H.rows) {
					atomicAdd((unsigned long long *)(H.rows + s), 1ULL);
				}
#pragma unroll
				for (int i = 0; i < 4; i++) {
					if (i < P.ninputs && H.A[i]) {
						uint64_t raw = *(const uint64_t *)(stage + P.in_off[i] + (size_t)r * 8);
						atomicAdd((unsigned long long *)(H.A[i] + s), (unsigned long long)(raw & 0xffffffffULL));
						uint64_t hi = ((P.in_signed >> i) & 1) ? (uint64_t)((int64_t)raw >> 32) : (raw >> 32);
						if (hi) {
							atomicAdd((unsigned long long *)(H.B[i] + s), (unsigned long long)hi);
						}
					}
				}
			}
			// deferred rows of the warp -> list, one atomic per warp
			__syncwarp();
			if (__any_sync(0xffffffffu, defer != 0)) {
				uint32_t n = __popc(defer), incl = n;
#pragma unroll
				for (int off = 1; off < 32; off <<= 1) {
					uint32_t v = __shfl_up_sync(0xffffffffu, incl, off);
					if (lane >= off) {
						incl += v;
					}
				}
				uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
				unsigned long long base = 0;
				if (lane == 0) {
					base = atomicAdd(&P.counters[0], (unsigned long long)total);
				}
				base = __shfl_sync(0xffffffffu, base, 0) + incl - n;
#pragma unroll
				for (int k = 0; k < HC_RB; k++) {
					if ((defer >> k) & 1) {
						P.deferred[base++] = (uint32_t)(row0 + rb0 + tid + k * HC_THREADS);
					}
				}
			}
		}
	});
}

// ------------------------------------------------------------------ SIMPLE shape, one row per thread
// The table accesses are random L2 round trips; what hides them is the NUMBER of independent rows in flight, not a
// staged input pipeline.  This variant has no shared memory and no tile loop: every thread takes one row at a time
// (grid-stride, coalesced direct loads of the narrow input columns), 32-48 resident warps per SM.  It is the shape of
// the atomics micro-benchmark (scripts/ubench/atomics.cu).
struct HcDirect {
	int nkeys, ninputs;
	const unsigned char *key_ptr[4];
	uint32_t key_width[4], key_shift[4], key_word[4];
	const uint64_t *in_ptr[8];
	uint32_t in_signed;
	uint64_t row_begin, row_end;
	uint32_t *deferred;
	unsigned long long *counters;
};

__device__ __forceinline__ uint64_t hc_load_col(const unsigned char *p, uint64_t row, uint32_t width) {
	// read-once input columns: streaming (evict-first) loads, so that they do not push the table out of L2
	switch (width) {
	case 1:
		return __ldcs(p + row);
	case 2:
		return __ldcs((const uint16_t *)p + row);
	case 4:
		return __ldcs((const uint32_t *)p + row);
	default:
		return __ldcs((const unsigned long long *)p + row);
	}
}

#define HC_DR 2 // rows per thread in flight (independent probe chains)
template <int KW, int NIN>
__global__ void __launch_bounds__(256, 4) agg_hc_direct_kernel(const __grid_constant__ HcDirect P, const __grid_constant__ HcView H) {
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	const uint64_t occ = H.occ_bit;
	const int lane = threadIdx.x & 31;
	const uint64_t n = P.row_end - P.row_begin;
	const uint64_t iters = (n + stride * HC_DR - 1) / (stride * HC_DR); // uniform trip count (warp-collective deferral)
	for (uint64_t it = 0; it < iters; it++) {
		uint64_t row[HC_DR], k0[HC_DR], k1[HC_DR], k2[HC_DR], slot[HC_DR];
		uint64_t raw[HC_DR][NIN];
		bool live[HC_DR], pend[HC_DR], defer[HC_DR];
#pragma unroll
		for (int q = 0; q < HC_DR; q++) {
			row[q] = P.row_begin + (it * HC_DR + q) * stride + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
			live[q] = row[q] < P.row_end;
			defer[q] = false;
			k0[q] = k1[q] = k2[q] = 0;
			slot[q] = 0;
			if (live[q]) {
#pragma unroll
				for (int j = 0; j < 4; j++) {
					if (j < P.nkeys) {
						uint64_t v = hc_load_col(P.key_ptr[j], row[q], P.key_width[j]) << P.key_shift[j];
						uint32_t wd = P.key_word[j];
						k0[q] |= wd == 0 ? v : 0;
						if (KW >= 2) {
							k1[q] |= wd == 1 ? v : 0;
						}
						if (KW >= 3) {
							k2[q] |= wd == 2 ? v : 0;
						}
					}
				}
#pragma unroll
				for (int i = 0; i < NIN; i++) {
					raw[q][i] = i < P.ninputs ? __ldcs((const unsigned long long *)P.in_ptr[i] + row[q]) : 0;
				}
				slot[q] = hc_hash_words(k0[q], k1[q], k2[q], KW) & H.mask;
			}
			pend[q] = live[q];
		}
		// probe chains of the thread's rows advance together: their L2 round trips overlap
		while (pend[0] || pend[HC_DR - 1]) {
			uint64_t w[HC_DR][3];
#pragma unroll
			for (int q = 0; q < HC_DR; q++) {
				if (pend[q]) {
					hc_load_keys<KW>(H, slot[q], w[q]);
				}
			}
#pragma unroll
			for (int q = 0; q < HC_DR; q++) {
				if (!pend[q]) {
					continue;
				}
				const uint64_t klast = KW == 1 ? k0[q] : (KW == 2 ? k1[q] : k2[q]);
				const uint64_t last = w[q][KW - 1];
				bool eq = last == (klast | occ);
				if (KW >= 2) {
					eq = eq && w[q][0] == k0[q];
				}
				if (KW >= 3) {
					eq = eq && w[q][1] == k1[q];
				}
				if (eq) {
					pend[q] = false;
				} else if (last == 0 || (last & H.lock_bit)) {
					slot[q] = hc_slow_path<KW>(H, k0[q], k1[q], k2[q], slot[q], w[q][0], w[q][1], w[q][2]);
					defer[q] = slot[q] == SLOT_DEFER;
					pend[q] = false;
				} else {
					slot[q] = (slot[q] + 1) & H.mask;
				}
			}
		}
#pragma unroll
		for (int q = 0; q < HC_DR; q++) {
			if (live[q] && !defer[q]) {
				if (H.rows) {
					atomicAdd((unsigned long long *)(H.rows + slot[q]), 1ULL);
				}
#pragma unroll
				for (int i = 0; i < NIN; i++) {
					if (i < P.ninputs && H.A[i]) {
						atomicAdd((unsigned long long *)(H.A[i] + slot[q]), (unsigned long long)(raw[q][i] & 0xffffffffULL));
						uint64_t hi = ((P.in_signed >> i) & 1) ? (uint64_t)((int64_t)raw[q][i] >> 32) : (raw[q][i] >> 32);
						if (hi) {
							atomicAdd((unsigned long long *)(H.B[i] + slot[q]), (unsigned long long)hi);
						}
					}
				}
			}
		}
		__syncwarp();
#pragma unroll
		for (int q = 0; q < HC_DR; q++) {
			uint32_t dm = __ballot_sync(0xffffffffu, defer[q]);
			if (dm) {
				unsigned long long base = 0;
				if (lane == 0) {
					base = atomicAdd(&P.counters[0], (unsigned long long)__popc(dm));
				}
				base = __shfl_sync(0xffffffffu, base, 0);
				if (defer[q]) {
					P.deferred[base + __popc(dm & ((1u << lane) - 1))] = (uint32_t)row[q];
				}
			}
		}
	}
}

// Same sink for row-id lists (the replay of deferred rows after the table grew) and for inputs the TMA front end does
// not take (dictionary / constant vectors, unaligned columns): rows == nullptr -> rows [row_begin, row_end) themselves.
template <int KW>
__global__ void __launch_bounds__(256)
    agg_hc_rows_kernel(HcView H, AggLayout L, KeyCols keys, AggCols ac, uint64_t row_begin, uint64_t row_end,
                       const uint32_t *__restrict__ rows, uint32_t *__restrict__ deferred, unsigned long long *counters) {
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	const uint64_t n = row_end - row_begin;
	const uint64_t iters = (n + stride - 1) / stride; // uniform trip count: the deferral append is a warp-collective
	for (uint64_t it = 0; it < iters; it++) {
		uint64_t i = row_begin + it * stride + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
		uint32_t drow = 0;
		int ndef = 0;
		if (i < row_end) {
			uint64_t row = rows ? rows[i] : i;
			uint64_t kw[KEY_WORDS_MAX];
			pack_key_row<false>(L, keys, row, kw);
			uint64_t slot = hc_hash(kw, KW) & H.mask, w[3];
			hc_load_keys<KW>(H, slot, w);
			uint64_t s = hc_find_or_create<KW>(H, kw, slot, w);
			if (s == SLOT_DEFER) {
				drow = (uint32_t)row;
				ndef = 1;
			} else {
				if (H.rows) {
					atomicAdd((unsigned long long *)(H.rows + s), 1ULL);
				}
				for (int a = 0; a < L.ninputs; a++) {
					const DCol &c = ac.c[a];
					uint64_t idx = col_index(c, row);
					if (col_valid_at(c, idx)) {
						hc_apply(H, L, s, a, col_load_raw(c, idx));
					}
				}
			}
		}
		__syncwarp();
		hc_defer_rows(deferred, &counters[0], &drow, ndef);
	}
}

// merge every group of the HC table into the generic table (which has been grown to hold them)
template <int KW>
__global__ void __launch_bounds__(256) agg_hc_flush_kernel(HcView H, uint64_t cap, AggTable T, AggLayout L, AggCols ac) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride) {
		uint64_t kw[KEY_WORDS_MAX] = {0, 0, 0, 0};
		uint64_t last = H.keys[s * HC_KWS(KW) + KW - 1];
		if (!last) {
			continue;
		}
		kw[KW - 1] = last & ~(H.occ_bit | H.lock_bit);
#pragma unroll
		for (int q = 0; q < KW - 1; q++) {
			kw[q] = H.keys[s * HC_KWS(KW) + q];
		}
		uint64_t gs = agg_find_or_create(T, L, hash_packed_key(L, kw), kw, ~0ULL);
		uint64_t *grow = T.slots + gs * (uint64_t)L.stride;
		// without a rows array no aggregate reads a count: rows only has to be non-zero ("the group exists")
		uint64_t rows = H.rows ? H.rows[s] : 1;
		atomicAdd((unsigned long long *)(grow + L.rows_off), (unsigned long long)rows);
		for (int i = 0; i < L.ninputs; i++) {
			if (ac.track_cnt[i]) {
				uint64_t c = H.cnt[i] ? H.cnt[i][s] : rows;
				if (c) {
					atomicAdd((unsigned long long *)(grow + L.cnt_off[i]), (unsigned long long)c);
				}
			}
			if (H.A[i]) {
				uint64_t lo, hi;
				hc_sum128(L.input_type[i], H.A[i][s], H.B[i][s], &lo, &hi);
				if (lo | hi) {
					atomic_add_128(grow + L.sum_off[i], grow + L.sum_off[i] + 1, lo, hi);
				}
			}
		}
	}
}

// Move the groups of the generic table (the adaptation probe's rows) INTO this table, so that afterwards every group
// lives here and finalize can read this table directly instead of merging it into the generic one.
template <int KW>
__global__ void __launch_bounds__(256)
    agg_hc_absorb_kernel(HcView H, AggLayout L, const uint64_t *slots, uint64_t capacity, AggCols ac,
                         unsigned long long *failed) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
		const uint64_t *row = slots + s * (uint64_t)L.stride;
		if (!row[0]) {
			continue;
		}
		uint64_t kw[KEY_WORDS_MAX] = {0, 0, 0, 0};
		for (int q = 0; q < KW; q++) {
			kw[q] = row[1 + q];
		}
		uint64_t slot = hc_hash(kw, KW) & H.mask, w[3];
		hc_load_keys<KW>(H, slot, w);
		uint64_t d = hc_find_or_create<KW>(H, kw, slot, w);
		if (d == SLOT_DEFER) {
			atomicAdd(failed, 1ULL);
			continue;
		}
		uint64_t rows = row[L.rows_off];
		if (H.rows) {
			atomicAdd((unsigned long long *)(H.rows + d), (unsigned long long)rows);
		}
		for (int i = 0; i < L.ninputs; i++) {
			if (H.cnt[i]) {
				atomicAdd((unsigned long long *)(H.cnt[i] + d), (unsigned long long)(ac.track_cnt[i] ? row[L.cnt_off[i]] : rows));
			}
			if (H.A[i]) {
				uint64_t lo = row[L.sum_off[i]], hi = row[L.sum_off[i] + 1];
				atomicAdd((unsigned long long *)(H.A[i] + d), (unsigned long long)(lo & 0xffffffffULL));
				uint64_t hp = (hi << 32) | (lo >> 32);
				if (hp) {
					atomicAdd((unsigned long long *)(H.B[i] + d), (unsigned long long)hp);
				}
			}
		}
	}
}

// finalize straight from this table (same output contract as agg_finalize_kernel of agg.cu; integer aggregates only)
template <int KW>
__global__ void __launch_bounds__(256)
    agg_hc_finalize_kernel(HcView H, uint64_t cap, AggLayout L, FinalizeOut out, unsigned long long *out_counter) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride) {
		uint64_t last = H.keys[s * HC_KWS(KW) + KW - 1];
		if (!last) {
			continue;
		}
		uint64_t kw[KEY_WORDS_MAX] = {0, 0, 0, 0};
		kw[KW - 1] = last & ~(H.occ_bit | H.lock_bit);
#pragma unroll
		for (int q = 0; q < KW - 1; q++) {
			kw[q] = H.keys[s * HC_KWS(KW) + q];
		}
		uint64_t g = atomicAdd(out_counter, 1ULL);
		write_keys(L, kw, g, out.key_data, out.key_valid);
		uint64_t rows = H.rows ? H.rows[s] : 1;
		for (int a = 0; a < L.naggs; a++) {
			int func = L.func[a], t = L.in_type[a], i = L.input[a];
			uint64_t cnt = i < 0 ? rows : (H.cnt[i] ? H.cnt[i][s] : rows);
			bool valid = cnt != 0;
			uint64_t lo = 0, hi = 0;
			if (i >= 0 && H.A[i]) {
				hc_sum128(t, H.A[i][s], H.B[i][s], &lo, &hi);
			}
			switch (func) {
			case B200_AGG_COUNT_STAR:
			case B200_AGG_COUNT:
				((uint64_t *)out.agg_data[a])[g] = cnt;
				valid = true;
				break;
			case B200_AGG_SUM:
				((uint64_t *)out.agg_data[a])[2 * g] = lo;
				((uint64_t *)out.agg_data[a])[2 * g + 1] = hi;
				break;
			case B200_AGG_SUM_NO_OVERFLOW:
				((uint64_t *)out.agg_data[a])[g] = lo;
				break;
			case B200_AGG_AVG:
				((uint64_t *)out.agg_data[a])[3 * g] = lo;
				((uint64_t *)out.agg_data[a])[3 * g + 1] = hi;
				((uint64_t *)out.agg_data[a])[3 * g + 2] = cnt;
				break;
			default:
				break;
			}
			if (!valid) {
				atomicAnd((unsigned long long *)&out.agg_valid[a][g >> 6], ~(1ULL << (g & 63)));
			}
		}
	}
}

// move every group into a larger HC table
template <int KW>
__global__ void __launch_bounds__(256) agg_hc_rehash_kernel(HcView O, uint64_t old_cap, HcView N, int ninputs) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < old_cap; s += stride) {
		uint64_t last = O.keys[s * HC_KWS(KW) + KW - 1];
		if (!last) {
			continue;
		}
		uint64_t kw[KEY_WORDS_MAX] = {0, 0, 0, 0};
		kw[KW - 1] = last & ~(O.occ_bit | O.lock_bit);
#pragma unroll
		for (int q = 0; q < KW - 1; q++) {
			kw[q] = O.keys[s * HC_KWS(KW) + q];
		}
		uint64_t pos = hc_hash(kw, KW) & N.mask;
		while (true) {
			unsigned long long old =
			    atomicCAS((unsigned long long *)&N.keys[pos * HC_KWS(KW) + KW - 1], 0ULL, (unsigned long long)last);
			if (old == 0ULL) {
				break;
			}
			pos = (pos + 1) & N.mask;
		}
#pragma unroll
		for (int q = 0; q < KW - 1; q++) {
			N.keys[pos * HC_KWS(KW) + q] = kw[q];
		}
		if (O.rows) {
			N.rows[pos] = O.rows[s];
		}
		for (int i = 0; i < ninputs; i++) {
			if (O.A[i]) {
				N.A[i][pos] = O.A[i][s];
				N.B[i][pos] = O.B[i][s];
			}
			if (O.cnt[i]) {
				N.cnt[i][pos] = O.cnt[i][s];
			}
		}
	}
}

// ------------------------------------------------------------------ host
#define HC_DISPATCH(kw, CALL)                                                                                          \
	do {                                                                                                               \
		if ((kw) == 3) {                                                                                               \
			constexpr int KW = 3;                                                                                      \
			CALL;                                                                                                      \
		} else if ((kw) == 2) {                                                                                        \
			constexpr int KW = 2;                                                                                      \
			CALL;                                                                                                      \
		} else {                                                                                                       \
			constexpr int KW = 1;                                                                                      \
			CALL;                                                                                                      \
		}                                                                                                              \
	} while (0)

int b200_agg_hc_eligible(const AggLayout &L) {
	if (L.key_words > 3 || L.nkeys > 6) {
		return B200_ERR_INVALID;
	}
	for (int i = 0; i < L.ninputs; i++) {
		if (!b200_type_is_integer(L.input_type[i]) || L.min_off[i] >= 0 || L.max_off[i] >= 0) {
			return B200_ERR_INVALID;
		}
	}
	return B200_OK;
}

static int hc_alloc(b200_ctx *ctx, const AggLayout &L, const bool *track_cnt, bool need_rows, uint64_t cap, AggHc *hc,
                    unsigned long long *count_dev) {
	int kw = L.key_words;
	size_t arrays = (size_t)HC_KWS(kw) + (need_rows ? 1 : 0);
	for (int i = 0; i < L.ninputs; i++) {
		arrays += (L.sum_off[i] >= 0 ? 2 : 0) + (track_cnt[i] ? 1 : 0);
	}
	size_t bytes = arrays * cap * 8;
	void *mem = nullptr;
	B200_TRY(b200_dev_alloc(ctx, bytes + 64, &mem));
	CUDA_TRY(cudaMemsetAsync(mem, 0, bytes, ctx->stream));
	memset(&hc->V, 0, sizeof(hc->V));
	uint64_t *p = (uint64_t *)mem;
	hc->V.keys = p;
	p += (size_t)HC_KWS(kw) * cap;
	if (need_rows) {
		hc->V.rows = p;
		p += cap;
	}
	// hot arrays first (A of every input, cnt of nullable inputs), the rarely touched high halves last
	for (int i = 0; i < L.ninputs; i++) {
		if (L.sum_off[i] >= 0) {
			hc->V.A[i] = p;
			p += cap;
		}
		if (track_cnt[i]) {
			hc->V.cnt[i] = p;
			p += cap;
		}
	}
	hc->hot_bytes = (size_t)((unsigned char *)p - (unsigned char *)mem); // (the rarely touched B arrays follow)
	hc->pinned_mem = nullptr;
	for (int i = 0; i < L.ninputs; i++) {
		if (L.sum_off[i] >= 0) {
			hc->V.B[i] = p;
			p += cap;
		}
	}
	hc->V.mask = cap - 1;
	hc->V.count = count_dev;
	// load factor <= 0.69, exact: a group is reserved in the CTA's shard before its slot is claimed
	hc->V.limit = (cap - cap / 4 - cap / 16) / HC_SHARDS;
	int sh = (L.null_off & 7) * 8;
	hc->V.occ_bit = 0x80ULL << sh;
	hc->V.lock_bit = 0x40ULL << sh;
	hc->kw = kw;
	hc->cap = cap;
	hc->mem = mem;
	hc->need_rows = need_rows;
	for (int i = 0; i < MAX_INPUTS; i++) {
		hc->track_cnt[i] = i < L.ninputs && track_cnt[i];
	}
	return B200_OK;
}

void b200_agg_hc_destroy(b200_ctx *ctx, AggHc *hc) {
	if (!hc) {
		return;
	}
	b200_dev_free(ctx, hc->mem);
	b200_dev_free(ctx, hc->V.count);
	delete hc;
}

uint64_t b200_agg_hc_capacity(const AggHc *hc) {
	return hc->cap;
}

__global__ void hc_count_kernel(const unsigned long long *shards, unsigned long long *out) {
	unsigned long long t = 0;
	for (int i = 0; i < HC_SHARDS; i++) {
		t += shards[i * 4];
	}
	*out = t;
}

// rebalance the shards after a rehash so that every CTA residue gets the same headroom again
__global__ void hc_spread_count_kernel(unsigned long long *shards) {
	unsigned long long t = 0;
	for (int i = 0; i < HC_SHARDS; i++) {
		t += shards[i * 4];
	}
	for (int i = 0; i < HC_SHARDS; i++) {
		shards[i * 4] = t / HC_SHARDS + ((unsigned long long)i < t % HC_SHARDS ? 1 : 0);
	}
}

int b200_agg_hc_groups(b200_ctx *ctx, AggHc *hc, uint64_t *groups) {
	unsigned long long *total = hc->V.count + HC_SHARDS * 4;
	hc_count_kernel<<<1, 1, 0, ctx->stream>>>(hc->V.count, total);
	ctx->launches++;
	CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 24, total, 8, cudaMemcpyDeviceToHost, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	CUDA_TRY(cudaGetLastError());
	ctx->d2h_bytes += 8;
	*groups = ctx->pinned_scratch[24];
	return B200_OK;
}

int b200_agg_hc_grow(b200_ctx *ctx, const AggLayout &L, AggHc *hc, uint64_t new_cap) {
	AggHc bigger = *hc;
	B200_TRY(hc_alloc(ctx, L, hc->track_cnt, hc->need_rows, new_cap, &bigger, hc->V.count));
	int grid = grid_for(hc->cap, 256, 4, ctx->sm_count * 8);
	HC_DISPATCH(hc->kw, (agg_hc_rehash_kernel<KW><<<grid, 256, 0, ctx->stream>>>(hc->V, hc->cap, bigger.V, L.ninputs)));
	hc_spread_count_kernel<<<1, 1, 0, ctx->stream>>>(hc->V.count);
	ctx->launches += 2;
	b200_dev_free(ctx, hc->mem);
	bigger.rows_sunk = hc->rows_sunk;
	*hc = bigger;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// does the table `hc` still match the aggregate's state configuration (nullable inputs may have appeared)?
bool b200_agg_hc_compatible(const AggHc *hc, const AggLayout &L, const bool *track_cnt) {
	for (int i = 0; i < L.ninputs; i++) {
		if (hc->track_cnt[i] != track_cnt[i]) {
			return false;
		}
	}
	return hc->rows_sunk < (1ULL << 31); // the 32-bit halves are summed in 64-bit words: merge before they could wrap
}

// Create the table (room for `groups_hint` groups at load <= 0.5) or grow an existing one to that size.
int b200_agg_hc_prepare(b200_ctx *ctx, AggHc **hc_io, const AggLayout &L, const bool *track_cnt, uint64_t groups_hint) {
	bool need_rows = false;
	for (int a = 0; a < L.naggs; a++) {
		need_rows = need_rows || L.func[a] == B200_AGG_COUNT_STAR || L.func[a] == B200_AGG_COUNT || L.func[a] == B200_AGG_AVG;
	}
	uint64_t want = HC_MIN_CAP;
	while (want < 2 * groups_hint) {
		want <<= 1;
	}
	if (!*hc_io) {
		AggHc *hc = new AggHc();
		memset((void *)hc, 0, sizeof(*hc));
		void *c = nullptr;
		int rc = b200_dev_alloc(ctx, (HC_SHARDS * 4 + 8) * 8, &c);
		if (rc == B200_OK) {
			cudaMemsetAsync(c, 0, (HC_SHARDS * 4 + 8) * 8, ctx->stream);
			rc = hc_alloc(ctx, L, track_cnt, need_rows, want, hc, (unsigned long long *)c);
		}
		if (rc != B200_OK) {
			b200_dev_free(ctx, c);
			delete hc;
			return rc;
		}
		*hc_io = hc;
		return B200_OK;
	}
	if ((*hc_io)->cap < want) {
		return b200_agg_hc_grow(ctx, L, *hc_io, want);
	}
	return B200_OK;
}

// Sink rows of the batch into the HC table; rows that find it at its limit are appended to `deferred`
// (count in counters[0]).  rows == nullptr: the row range [row_begin, row_end) through the TMA-staged kernel when
// `staged` (flat, aligned columns; row_begin a multiple of the tile), else through the generic kernel;
// rows != nullptr: the row ids rows[row_begin .. row_end).
int b200_agg_hc_sink(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const KeyCols &keys, const AggCols &ac, bool staged,
                     const uint32_t *rows, uint64_t row_begin, uint64_t row_end, uint32_t *deferred,
                     unsigned long long *counters) {
	uint64_t n = row_end - row_begin;
	if (n == 0) {
		return B200_OK;
	}
	// keep the hot arrays of a table that fits three quarters of L2 in the persisting part of L2 while rows stream past
	// (opt-in, B200_HC_L2_PIN=1: pinning a table that outgrows the window slows the sink down; the effect on H100 is
	// not measured)
	if (getenv("B200_HC_L2_PIN") && hc->pinned_mem != hc->mem && hc->hot_bytes <= ctx->l2_size / 4 * 3 &&
	    !getenv("B200_NO_L2_PIN")) {
		b200_l2_pin(ctx, hc->mem, hc->hot_bytes);
		hc->pinned_mem = hc->mem;
	}
	if (rows || !staged) {
		int grid = grid_for(n, 256, 4, ctx->sm_count * 8);
		HC_DISPATCH(hc->kw, (agg_hc_rows_kernel<KW><<<grid, 256, 0, ctx->stream>>>(hc->V, L, keys, ac, row_begin, row_end, rows, deferred, counters)));
		ctx->launches++;
		if (!rows) {
			hc->rows_sunk += n;
		}
		CUDA_TRY(cudaGetLastError());
		return B200_OK;
	}
	TileArgs A;
	memset(&A, 0, sizeof(A));
	A.L = L;
	A.keys = keys;
	A.ac = ac;
	A.row_begin = row_begin;
	A.row_end = row_end;
	A.deferred = deferred;
	A.counters = counters;
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
	bool ok = true;
	for (int j = 0; j < L.nkeys; j++) {
		A.sm.key_data[j] = add(keys.c[j].data, b200_type_size(keys.c[j].type));
		A.sm.key_valid[j] = keys.c[j].validity ? add(keys.c[j].validity, 0) : -1;
		ok = ok && A.sm.key_data[j] >= 0 && (!keys.c[j].validity || A.sm.key_valid[j] >= 0);
	}
	for (int i = 0; i < L.ninputs; i++) {
		A.sm.in_data[i] = add(ac.c[i].data, b200_type_size(ac.c[i].type));
		A.sm.in_valid[i] = ac.c[i].validity ? add(ac.c[i].validity, 0) : -1;
		ok = ok && A.sm.in_data[i] >= 0 && (!ac.c[i].validity || A.sm.in_valid[i] >= 0);
	}
	if (!ok) {
		b200_set_error("agg hc path: too many staged columns");
		return B200_ERR_INVALID;
	}
	tile_cols_finish(&A.tc, AT_TILE);
	A.stages = 3;
	while (A.stages > 2 && (size_t)A.stages * A.tc.stage_bytes > 100 * 1024) {
		A.stages--;
	}
	size_t smem = (size_t)A.stages * A.tc.stage_bytes;
	if (smem > 200 * 1024) {
		b200_set_error("agg hc path: rows too wide for the staging tile");
		return B200_ERR_INVALID;
	}
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(agg_hc_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		attr_set = true;
	}
	uint64_t ntiles = (n + AT_TILE - 1) / AT_TILE;
	// SIMPLE: integer keys without NULLs + 8-byte integer inputs without NULLs, cnt not tracked
	HcKeyDesc D;
	memset(&D, 0, sizeof(D));
	bool simple = true;
	D.nkeys = L.nkeys;
	D.ninputs = L.ninputs;
	for (int j = 0; j < L.nkeys; j++) {
		simple = simple && b200_type_is_integer(L.key_type[j]) && !keys.c[j].validity;
		D.smem_off[j] = A.tc.c[A.sm.key_data[j]].smem_off;
		D.width[j] = (uint32_t)b200_type_size(L.key_type[j]);
		D.word[j] = (uint32_t)(L.key_off[j] >> 3);
		D.shift[j] = (uint32_t)((L.key_off[j] & 7) * 8);
	}
	for (int i = 0; i < L.ninputs; i++) {
		simple = simple && (L.input_type[i] == B200_INT64 || L.input_type[i] == B200_UINT64) && !ac.c[i].validity &&
		         !hc->track_cnt[i];
		D.in_off[i] = A.tc.c[A.sm.in_data[i]].smem_off;
	}
	int per_sm = 0;
	cudaError_t oe = cudaSuccess;
	if (simple && L.nkeys <= 4 && L.ninputs <= 8 && !getenv("B200_HC_TILE") && !getenv("B200_HC_GENERIC")) {
		HcDirect P;
		memset(&P, 0, sizeof(P));
		P.nkeys = L.nkeys;
		P.ninputs = L.ninputs;
		for (int j = 0; j < L.nkeys; j++) {
			P.key_ptr[j] = (const unsigned char *)keys.c[j].data;
			P.key_width[j] = D.width[j];
			P.key_shift[j] = D.shift[j];
			P.key_word[j] = D.word[j];
		}
		for (int i = 0; i < L.ninputs; i++) {
			P.in_ptr[i] = (const uint64_t *)ac.c[i].data;
			P.in_signed |= (L.input_type[i] == B200_INT64 ? 1u : 0u) << i;
		}
		P.row_begin = row_begin;
		P.row_end = row_end;
		P.deferred = deferred;
		P.counters = counters;
		int dgrid = grid_for(n, 256, 4, ctx->sm_count * 8);
		if (L.ninputs <= 1) {
			HC_DISPATCH(hc->kw, (agg_hc_direct_kernel<KW, 1><<<dgrid, 256, 0, ctx->stream>>>(P, hc->V)));
		} else if (L.ninputs <= 2) {
			HC_DISPATCH(hc->kw, (agg_hc_direct_kernel<KW, 2><<<dgrid, 256, 0, ctx->stream>>>(P, hc->V)));
		} else if (L.ninputs <= 4) {
			HC_DISPATCH(hc->kw, (agg_hc_direct_kernel<KW, 4><<<dgrid, 256, 0, ctx->stream>>>(P, hc->V)));
		} else {
			HC_DISPATCH(hc->kw, (agg_hc_direct_kernel<KW, 8><<<dgrid, 256, 0, ctx->stream>>>(P, hc->V)));
		}
		ctx->launches++;
		hc->rows_sunk += n;
		CUDA_TRY(cudaGetLastError());
		return B200_OK;
	}
	if (simple && L.nkeys <= 4 && L.ninputs <= 4 && !getenv("B200_HC_GENERIC")) {
		static bool sattr = false;
		if (!sattr) {
			CUDA_TRY(cudaFuncSetAttribute(agg_hc_simple_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
			CUDA_TRY(cudaFuncSetAttribute(agg_hc_simple_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
			CUDA_TRY(cudaFuncSetAttribute(agg_hc_simple_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
			sattr = true;
		}
		HcSimple P;
		memset(&P, 0, sizeof(P));
		P.tc = A.tc;
		P.stages = A.stages;
		P.nkeys = L.nkeys;
		P.ninputs = L.ninputs;
		for (int j = 0; j < L.nkeys; j++) {
			P.key_off[j] = D.smem_off[j];
			P.key_width[j] = D.width[j];
			P.key_shift[j] = D.shift[j];
			P.key_word[j] = D.word[j];
		}
		for (int i = 0; i < L.ninputs; i++) {
			P.in_off[i] = D.in_off[i];
			P.in_signed |= (L.input_type[i] == B200_INT64 ? 1u : 0u) << i;
		}
		P.row_begin = row_begin;
		P.row_end = row_end;
		P.deferred = deferred;
		P.counters = counters;
		HC_DISPATCH(hc->kw, (oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, agg_hc_simple_kernel<KW>, HC_THREADS + 32, smem)));
		CUDA_TRY(oe);
		per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
		uint64_t mg = (uint64_t)ctx->sm_count * per_sm;
		unsigned g = (unsigned)(ntiles < mg ? ntiles : mg);
		HC_DISPATCH(hc->kw, (agg_hc_simple_kernel<KW><<<g, HC_THREADS + 32, smem, ctx->stream>>>(P, hc->V)));
		ctx->launches++;
		hc->rows_sunk += n;
		CUDA_TRY(cudaGetLastError());
		return B200_OK;
	}
	HC_DISPATCH(hc->kw, (oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, agg_hc_kernel<KW, false>, HC_THREADS + 32, smem)));
	CUDA_TRY(oe);
	per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
	uint64_t max_grid = (uint64_t)ctx->sm_count * per_sm;
	unsigned grid = (unsigned)(ntiles < max_grid ? ntiles : max_grid);
	HC_DISPATCH(hc->kw, (agg_hc_kernel<KW, false><<<grid, HC_THREADS + 32, smem, ctx->stream>>>(A, hc->V, D)));
	ctx->launches++;
	hc->rows_sunk += n;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

int b200_agg_hc_flush(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const AggTable &T, const AggCols &ac) {
	int grid = grid_for(hc->cap, 256, 4, ctx->sm_count * 8);
	HC_DISPATCH(hc->kw, (agg_hc_flush_kernel<KW><<<grid, 256, 0, ctx->stream>>>(hc->V, hc->cap, T, L, ac)));
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// Empty the generic table's groups into this one (the caller re-initialises the generic table afterwards).
int b200_agg_hc_absorb(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const uint64_t *slots, uint64_t capacity,
                       const bool *track_cnt) {
	AggCols ac;
	memset(&ac, 0, sizeof(ac));
	for (int i = 0; i < L.ninputs; i++) {
		ac.track_cnt[i] = track_cnt[i];
	}
	unsigned long long *failed = hc->V.count + HC_SHARDS * 4 + 1;
	CUDA_TRY(cudaMemsetAsync(failed, 0, 8, ctx->stream));
	int grid = grid_for(capacity, 256, 4, ctx->sm_count * 8);
	HC_DISPATCH(hc->kw, (agg_hc_absorb_kernel<KW><<<grid, 256, 0, ctx->stream>>>(hc->V, L, slots, capacity, ac, failed)));
	ctx->launches++;
	CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 25, failed, 8, cudaMemcpyDeviceToHost, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	CUDA_TRY(cudaGetLastError());
	if (ctx->pinned_scratch[25]) {
		b200_set_error("agg hc path: the table had no room for the generic table's groups");
		return B200_ERR_CAPACITY;
	}
	return B200_OK;
}

int b200_agg_hc_finalize(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const FinalizeOut &fo, unsigned long long *out_counter) {
	int grid = grid_for(hc->cap, 256, 4, ctx->sm_count * 8);
	HC_DISPATCH(hc->kw, (agg_hc_finalize_kernel<KW><<<grid, 256, 0, ctx->stream>>>(hc->V, hc->cap, L, fo, out_counter)));
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// the sink of a batch is over: give the persisting L2 lines back
void b200_agg_hc_unpin(b200_ctx *ctx, AggHc *hc) {
	if (hc && hc->pinned_mem) {
		b200_l2_unpin(ctx);
		hc->pinned_mem = nullptr;
	}
}
