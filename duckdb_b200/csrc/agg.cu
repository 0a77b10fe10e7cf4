// K6 groupby_aggregate (host side + global-table path) + K7 aggregate_combine + finalize.
// Reference semantics: GroupedAggregateHashTable::FindOrCreateGroupsInternal / UpdateAggregates / Combine
// (src/execution/aggregate_hashtable.cpp:803-977,688-722,1168-1197), RowOperations::UpdateStates /
// CombineStates / FinalizeStates (src/common/row_operations/row_aggregate.cpp:52-64,120-150),
// sum / avg / count / min / max state arithmetic (extension/core_functions/aggregate/distributive/sum.cpp,
// include/core_functions/aggregate/sum_helpers.hpp:107-215, algebraic/avg.cpp:84-140).
// Design (GPU-first, not the reference's pointer-table + row store): ONE open-addressing table whose slot
// row holds [tag | packed key | shared aggregate states], so a row update touches one or two 32-byte sectors.
// Three sink paths, chosen adaptively per aggregate (the analogue of RadixPartitionedHashTable::DecideAdaptation,
// radix_partitioned_hashtable.cpp:533-571):
//   FAST   <= 16 groups per CTA : thread-private accumulators in shared memory      (agg_tile.cu)
//   MID    <= ~1-2 K groups     : per-CTA shared-memory hash table, 32-bit ATOMS    (agg_tile.cu)
//   GLOBAL anything             : atomics on the global table                       (this file)
#include "agg.cuh"
#include <cstring>
#include <cstdlib>
#include <vector>

int b200_fill_keycols(const b200_batch *b, const int *cols, int n, KeyCols *out, const char *who);

// agg_tile.cu
int b200_agg_tile_eligible(const AggLayout &L, const KeyCols &keys, const AggCols &ac);
uint64_t b200_agg_tile_headroom(int mode, int sm_count);
int b200_agg_tile_sink(b200_ctx *ctx, int mode, int slots_hint, const AggLayout &L, const AggTable &T,
                       const KeyCols &keys, const AggCols &ac, uint64_t row_begin, uint64_t row_end,
                       uint32_t *deferred, unsigned long long *counters, const PrivDirect *direct);
// agg_priv.cu
bool b200_agg_priv_build_direct(const AggLayout &L, const uint64_t *kw0, int ngroups, int max_slots, PrivDirect *PD,
                                std::vector<uint8_t> *out_tables);

// agg_priv.cu: groups per CTA the thread-private shared-memory path can hold for this layout (0 = not eligible)
int b200_agg_priv_capacity(const AggLayout &L);

// agg_hc.cu: the L2-first structure-of-arrays table for high cardinalities
struct AggHc;
int b200_agg_hc_eligible(const AggLayout &L);
int b200_agg_hc_prepare(b200_ctx *ctx, AggHc **hc_io, const AggLayout &L, const bool *track_cnt, uint64_t groups_hint);
bool b200_agg_hc_compatible(const AggHc *hc, const AggLayout &L, const bool *track_cnt);
uint64_t b200_agg_hc_capacity(const AggHc *hc);
int b200_agg_hc_groups(b200_ctx *ctx, AggHc *hc, uint64_t *groups);
int b200_agg_hc_grow(b200_ctx *ctx, const AggLayout &L, AggHc *hc, uint64_t new_cap);
int b200_agg_hc_sink(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const KeyCols &keys, const AggCols &ac, bool staged,
                     const uint32_t *rows, uint64_t row_begin, uint64_t row_end, uint32_t *deferred,
                     unsigned long long *counters);
int b200_agg_hc_flush(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const AggTable &T, const AggCols &ac);
int b200_agg_hc_absorb(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const uint64_t *slots, uint64_t capacity,
                       const bool *track_cnt);
int b200_agg_hc_finalize(b200_ctx *ctx, AggHc *hc, const AggLayout &L, const FinalizeOut &fo, unsigned long long *out_counter);
void b200_agg_hc_destroy(b200_ctx *ctx, AggHc *hc);
void b200_agg_hc_unpin(b200_ctx *ctx, AggHc *hc);

// sink paths in escalation order (b200_agg_sink's adaptation picks one from the group count of a probe chunk)
enum { PATH_FAST4 = 0, PATH_FAST = 1, PATH_PRIV = 2, PATH_MID = 3, PATH_HC = 4, PATH_GLOBAL = 5 };

struct b200_agg {
	b200_ctx *ctx;
	AggLayout L;
	uint64_t capacity;
	uint64_t *slots;
	unsigned long long *count;    // device counter: groups
	unsigned long long *counters; // device: [0] deferred rows, [1] rows that missed the shared-memory path, [2] scratch
	bool track_cnt[MAX_INPUTS];   // sticky: input i has been seen with a validity mask
	int path;                     // current sink path
	int path_groups;              // group count the path was chosen for (sizes the PRIV slots)
	uint64_t path_groups_hc;      // ... uncapped (initial size of the high-cardinality table)
	bool path_decided;
	uint64_t rows_seen;
	AggHc *hc;                    // high-cardinality front-end table (merged into `slots` before any read-out)
	bool aos_empty;               // every group lives in `hc` (the generic table was emptied into it): finalize reads hc
	PrivDirect priv_direct;       // PRIV path: direct slot addressing tables (nslots == 0: directory lookup instead)
	void *priv_direct_dev;
};

// packed key word 0 of every group (PRIV's direct addressing tables are built from them)
__global__ void agg_list_keys_kernel(const uint64_t *slots, uint64_t capacity, int stride, uint64_t *out, unsigned int max_out,
                                     unsigned int *counter) {
	uint64_t step = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += step) {
		const uint64_t *row = slots + s * (uint64_t)stride;
		if (row[0]) {
			unsigned int i = atomicAdd(counter, 1u);
			if (i < max_out) {
				out[i] = row[1];
			}
		}
	}
}

// ------------------------------------------------------------------ kernels
__global__ void agg_init_kernel(uint64_t *slots, uint64_t capacity, AggLayout L) {
	uint64_t total = capacity * (uint64_t)L.stride;
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
		int w = (int)(i % (uint64_t)L.stride);
		uint64_t v = 0;
		for (int a = 0; a < L.ninputs; a++) {
			if (L.min_off[a] >= 0 && w == L.min_off[a]) {
				v = ~0ULL;
			}
		}
		slots[i] = v;
	}
}

// rows = nullptr: process rows [row_begin, row_end); else rows[row_begin..row_end) are row ids
__global__ void __launch_bounds__(256)
    agg_sink_kernel(AggTable T, AggLayout L, KeyCols keys, AggCols ac, uint64_t row_begin, uint64_t row_end,
                    const uint32_t *__restrict__ rows, uint32_t *__restrict__ deferred,
                    unsigned long long *__restrict__ counters) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = row_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_end; i += stride) {
		uint64_t row = rows ? rows[i] : i;
		uint64_t kw[KEY_WORDS_MAX];
		uint64_t h = pack_key_row(L, keys, row, kw);
		// issue the input loads before the (dependent, random) table access
		uint64_t raw[MAX_INPUTS];
		uint32_t validbits = 0;
#pragma unroll
		for (int a = 0; a < MAX_INPUTS; a++) {
			if (a < L.ninputs) {
				const DCol &c = ac.c[a];
				uint64_t idx = col_index(c, row);
				validbits |= (col_valid_at(c, idx) ? 1u : 0u) << a;
				raw[a] = col_load_raw(c, idx);
			}
		}
		uint64_t slot = agg_find_or_create(T, L, h, kw);
		if (slot == SLOT_DEFER) {
			unsigned long long d = atomicAdd(&counters[0], 1ULL);
			deferred[d] = (uint32_t)row;
			continue;
		}
		uint64_t *srow = T.slots + slot * (uint64_t)L.stride;
		atomicAdd((unsigned long long *)(srow + L.rows_off), 1ULL);
#pragma unroll
		for (int a = 0; a < MAX_INPUTS; a++) {
			if (a < L.ninputs && ((validbits >> a) & 1)) {
				agg_apply_input(L, a, srow, raw[a], ac.track_cnt[a]);
			}
		}
	}
}

// cnt(x) starts being tracked: bring it up to date (cnt == rows for every existing group)
__global__ void agg_fix_cnt_kernel(uint64_t *slots, uint64_t capacity, AggLayout L, int input) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
		uint64_t *row = slots + s * (uint64_t)L.stride;
		if (row[0]) {
			row[L.cnt_off[input]] = row[L.rows_off];
		}
	}
}

// move every occupied slot of the old table into the new (larger) one
__global__ void __launch_bounds__(256)
    agg_rehash_kernel(const uint64_t *old_slots, uint64_t old_cap, AggTable T, AggLayout L) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < old_cap; s += stride) {
		const uint64_t *orow = old_slots + s * (uint64_t)L.stride;
		uint64_t tag = orow[0];
		if (!tag) {
			continue;
		}
		uint64_t pos = orow[L.hash_off] & T.mask;
		while (true) {
			uint64_t *nrow = T.slots + pos * (uint64_t)L.stride;
			unsigned long long old = atomicCAS((unsigned long long *)nrow, 0ULL, (unsigned long long)tag);
			if (old == 0) {
				for (int w = 1; w < L.stride; w++) {
					nrow[w] = orow[w];
				}
				break;
			}
			pos = (pos + 1) & T.mask;
		}
	}
}

__global__ void __launch_bounds__(256)
    agg_finalize_kernel(const uint64_t *slots, uint64_t capacity, AggLayout L, FinalizeOut out,
                        unsigned long long *out_counter) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
		const uint64_t *row = slots + s * (uint64_t)L.stride;
		if (!row[0]) {
			continue;
		}
		uint64_t g = atomicAdd(out_counter, 1ULL);
		write_keys(L, row + 1, g, out.key_data, out.key_valid);
		uint64_t rows = row[L.rows_off];
		for (int a = 0; a < L.naggs; a++) {
			int func = L.func[a], t = L.in_type[a], i = L.input[a];
			uint64_t cnt = i < 0 ? rows : (out.track_cnt[i] ? row[L.cnt_off[i]] : rows);
			bool valid = cnt != 0;
			switch (func) {
			case B200_AGG_COUNT_STAR:
			case B200_AGG_COUNT:
				((uint64_t *)out.agg_data[a])[g] = cnt;
				valid = true;
				break;
			case B200_AGG_SUM:
				if (b200_type_is_float(t)) {
					((uint64_t *)out.agg_data[a])[g] = row[L.sum_off[i]];
				} else {
					((uint64_t *)out.agg_data[a])[2 * g] = row[L.sum_off[i]];
					((uint64_t *)out.agg_data[a])[2 * g + 1] = row[L.sum_off[i] + 1];
				}
				break;
			case B200_AGG_SUM_NO_OVERFLOW:
				((uint64_t *)out.agg_data[a])[g] = row[L.sum_off[i]];
				break;
			case B200_AGG_AVG:
				if (b200_type_is_float(t)) {
					double sum = __longlong_as_double((long long)row[L.sum_off[i]]);
					((double *)out.agg_data[a])[g] = valid ? sum / (double)cnt : 0.0;
				} else {
					// raw triple; the host finishes with long double like IntegerAverageOperationHugeint::Finalize
					((uint64_t *)out.agg_data[a])[3 * g] = row[L.sum_off[i]];
					((uint64_t *)out.agg_data[a])[3 * g + 1] = row[L.sum_off[i] + 1];
					((uint64_t *)out.agg_data[a])[3 * g + 2] = cnt;
				}
				break;
			case B200_AGG_MIN:
				store_raw(out.agg_data[a], t, g, valid ? decode_ordered(t, row[L.min_off[i]]) : 0);
				break;
			case B200_AGG_MAX:
				store_raw(out.agg_data[a], t, g, valid ? decode_ordered(t, row[L.max_off[i]]) : 0);
				break;
			}
			if (!valid) {
				atomicAnd((unsigned long long *)&out.agg_valid[a][g >> 6], ~(1ULL << (g & 63)));
			}
		}
	}
}

// export: keys as typed columns, physical states as raw uint64 columns, in slot-row order
// [rows][input 0: cnt, sum.., min, max][input 1: ...]
#define MAX_STATE_COLS (1 + MAX_INPUTS * 5)
struct ExportOut {
	void *key_data[MAX_KEYS];
	uint64_t *key_valid[MAX_KEYS];
	uint64_t *state_cols[MAX_STATE_COLS];
	bool track_cnt[MAX_INPUTS];
};

struct StateMap {
	int n;
	int off[MAX_STATE_COLS];
	int cnt_input[MAX_STATE_COLS]; // input index when the column is a cnt column, else -1
};

static void state_map(const AggLayout &L, StateMap *sm) {
	int n = 0;
	sm->off[n] = L.rows_off;
	sm->cnt_input[n++] = -1;
	for (int i = 0; i < L.ninputs; i++) {
		sm->off[n] = L.cnt_off[i];
		sm->cnt_input[n++] = i;
		if (L.sum_off[i] >= 0) {
			sm->off[n] = L.sum_off[i];
			sm->cnt_input[n++] = -1;
			if (!b200_type_is_float(L.input_type[i])) {
				sm->off[n] = L.sum_off[i] + 1;
				sm->cnt_input[n++] = -1;
			}
		}
		if (L.min_off[i] >= 0) {
			sm->off[n] = L.min_off[i];
			sm->cnt_input[n++] = -1;
		}
		if (L.max_off[i] >= 0) {
			sm->off[n] = L.max_off[i];
			sm->cnt_input[n++] = -1;
		}
	}
	sm->n = n;
}

__global__ void __launch_bounds__(256)
    agg_export_kernel(const uint64_t *slots, uint64_t capacity, AggLayout L, ExportOut out, StateMap sm,
                      unsigned long long *out_counter) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
		const uint64_t *row = slots + s * (uint64_t)L.stride;
		if (!row[0]) {
			continue;
		}
		uint64_t g = atomicAdd(out_counter, 1ULL);
		write_keys(L, row + 1, g, out.key_data, out.key_valid);
		for (int c = 0; c < sm.n; c++) {
			uint64_t v = row[sm.off[c]];
			if (sm.cnt_input[c] >= 0 && !out.track_cnt[sm.cnt_input[c]]) {
				v = row[L.rows_off]; // cnt(x) == rows while x has never been nullable
			}
			out.state_cols[c][g] = v;
		}
	}
}

struct StateCols {
	const uint64_t *c[MAX_STATE_COLS];
};

__global__ void __launch_bounds__(256)
    agg_combine_kernel(AggTable T, AggLayout L, KeyCols keys, StateCols sc, uint64_t row_begin, uint64_t row_end,
                       const uint32_t *__restrict__ rows, uint32_t *__restrict__ deferred,
                       unsigned long long *__restrict__ counters) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = row_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_end; i += stride) {
		uint64_t row = rows ? rows[i] : i;
		uint64_t kw[KEY_WORDS_MAX];
		uint64_t h = pack_key_row(L, keys, row, kw);
		uint64_t slot = agg_find_or_create(T, L, h, kw);
		if (slot == SLOT_DEFER) {
			unsigned long long d = atomicAdd(&counters[0], 1ULL);
			deferred[d] = (uint32_t)row;
			continue;
		}
		uint64_t *srow = T.slots + slot * (uint64_t)L.stride;
		int c = 0;
		atomicAdd((unsigned long long *)(srow + L.rows_off), (unsigned long long)sc.c[c++][row]);
		for (int a = 0; a < L.ninputs; a++) {
			uint64_t cnt = sc.c[c++][row];
			atomicAdd((unsigned long long *)(srow + L.cnt_off[a]), (unsigned long long)cnt);
			if (L.sum_off[a] >= 0) {
				if (b200_type_is_float(L.input_type[a])) {
					double d = __longlong_as_double((long long)sc.c[c++][row]);
					if (cnt) {
						atomicAdd((double *)(srow + L.sum_off[a]), d);
					}
				} else {
					uint64_t lo = sc.c[c][row], hi = sc.c[c + 1][row];
					c += 2;
					atomic_add_128(srow + L.sum_off[a], srow + L.sum_off[a] + 1, lo, hi);
				}
			}
			if (L.min_off[a] >= 0) {
				atomicMin((unsigned long long *)(srow + L.min_off[a]), (unsigned long long)sc.c[c++][row]);
			}
			if (L.max_off[a] >= 0) {
				atomicMax((unsigned long long *)(srow + L.max_off[a]), (unsigned long long)sc.c[c++][row]);
			}
		}
	}
}


// ------------------------------------------------------------------ packed partial states (multi-GPU combine)
// One contiguous device buffer of uint64 words per rank, fixed size for a given max_groups, so that ONE
// all-gather moves every rank's partial aggregate and nothing has to be read back by the host:
//   word 0 = groups exported (<= max_groups), word 1 = flags (bit 0: the table held more than max_groups groups)
//   then (nkeys + 1 + nstate) columns of max_groups words: key j as its canonical 64-bit bits (sign-extended
//   integers, float / double BIT PATTERNS - never a value cast), the per-group NULL-key bits, the raw state columns
//   of b200_agg_export_states.
__global__ void __launch_bounds__(256)
    agg_export_packed_kernel(const uint64_t *slots, uint64_t capacity, AggLayout L, StateMap sm, ExportOut eo,
                             uint64_t *dst, uint64_t max_groups, unsigned long long *out_counter) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
		const uint64_t *row = slots + s * (uint64_t)L.stride;
		if (!row[0]) {
			continue;
		}
		uint64_t g = atomicAdd(out_counter, 1ULL);
		if (g >= max_groups) {
			continue;
		}
		uint64_t *col = dst + 2;
		uint64_t nullbits = 0;
		for (int j = 0; j < L.nkeys; j++) {
			bool is_null;
			uint64_t bits = unpack_key_field(L, row + 1, j, &is_null);
			col[g] = is_null ? 0 : bits;
			nullbits |= (uint64_t)(is_null ? 1 : 0) << j;
			col += max_groups;
		}
		col[g] = nullbits;
		col += max_groups;
		for (int c = 0; c < sm.n; c++) {
			uint64_t v = row[sm.off[c]];
			if (sm.cnt_input[c] >= 0 && !eo.track_cnt[sm.cnt_input[c]]) {
				v = row[L.rows_off];
			}
			col[g] = v;
			col += max_groups;
		}
	}
}

__global__ void agg_packed_header_kernel(uint64_t *dst, uint64_t max_groups, const unsigned long long *out_counter) {
	uint64_t g = *out_counter;
	dst[0] = g < max_groups ? g : max_groups;
	dst[1] = g > max_groups ? 1 : 0;
}

// combine nranks packed buffers (words_per_rank apart) into the table; counters[3] |= 1 when a buffer overflowed
__global__ void __launch_bounds__(128)
    agg_combine_packed_kernel(AggTable T, AggLayout L, StateMap sm, const uint64_t *src, uint64_t words_per_rank,
                              int nranks, uint64_t max_groups, unsigned long long *counters) {
	for (int r = blockIdx.x; r < nranks; r += gridDim.x) {
		const uint64_t *base = src + (uint64_t)r * words_per_rank;
		uint64_t ng = base[0];
		if (base[1] & 1) {
			if (threadIdx.x == 0) {
				atomicOr(&counters[3], 1ULL);
			}
			continue;
		}
		for (uint64_t g = threadIdx.x; g < ng && g < max_groups; g += blockDim.x) {
			const uint64_t *col = base + 2;
			uint64_t kw[KEY_WORDS_MAX] = {0, 0, 0, 0};
			uint64_t nullbits = col[(uint64_t)L.nkeys * max_groups + g];
			for (int j = 0; j < L.nkeys; j++) {
				if (!((nullbits >> j) & 1)) {
					pack_field(kw, L.key_off[j], key_field_bits(L.key_type[j], col[(uint64_t)j * max_groups + g]));
				}
			}
			pack_field(kw, L.null_off, nullbits & 0xff);
			col += (uint64_t)(L.nkeys + 1) * max_groups;
			uint64_t slot = agg_find_or_create(T, L, hash_packed_key(L, kw), kw, ~0ULL);
			uint64_t *srow = T.slots + slot * (uint64_t)L.stride;
			int c = 0;
			atomicAdd((unsigned long long *)(srow + L.rows_off), (unsigned long long)col[(uint64_t)(c++) * max_groups + g]);
			for (int a = 0; a < L.ninputs; a++) {
				uint64_t cnt = col[(uint64_t)(c++) * max_groups + g];
				atomicAdd((unsigned long long *)(srow + L.cnt_off[a]), (unsigned long long)cnt);
				if (L.sum_off[a] >= 0) {
					if (b200_type_is_float(L.input_type[a])) {
						double d = __longlong_as_double((long long)col[(uint64_t)(c++) * max_groups + g]);
						if (cnt) {
							atomicAdd((double *)(srow + L.sum_off[a]), d);
						}
					} else {
						uint64_t lo = col[(uint64_t)c * max_groups + g], hi = col[(uint64_t)(c + 1) * max_groups + g];
						c += 2;
						atomic_add_128(srow + L.sum_off[a], srow + L.sum_off[a] + 1, lo, hi);
					}
				}
				if (L.min_off[a] >= 0) {
					atomicMin((unsigned long long *)(srow + L.min_off[a]), (unsigned long long)col[(uint64_t)(c++) * max_groups + g]);
				}
				if (L.max_off[a] >= 0) {
					atomicMax((unsigned long long *)(srow + L.max_off[a]), (unsigned long long)col[(uint64_t)(c++) * max_groups + g]);
				}
			}
		}
	}
}

__global__ void fill_u64_kernel3(uint64_t *p, uint64_t words, uint64_t v) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) {
		p[i] = v;
	}
}

// ------------------------------------------------------------------ host side
static uint64_t next_pow2(uint64_t v) {
	uint64_t p = 1;
	while (p < v) {
		p <<= 1;
	}
	return p;
}

static int agg_alloc_table(b200_agg *agg, uint64_t capacity, uint64_t **out_slots) {
	void *p = nullptr;
	size_t bytes = (size_t)capacity * agg->L.stride * 8;
	B200_TRY(b200_dev_alloc(agg->ctx, bytes, &p));
	int grid = grid_for(capacity * agg->L.stride, 256, 4, agg->ctx->sm_count * 8);
	agg_init_kernel<<<grid, 256, 0, agg->ctx->stream>>>((uint64_t *)p, capacity, agg->L);
	agg->ctx->launches++;
	*out_slots = (uint64_t *)p;
	return B200_OK;
}

static AggTable agg_table(b200_agg *agg) {
	AggTable T;
	T.slots = agg->slots;
	T.mask = agg->capacity - 1;
	T.count = agg->count;
	T.limit = agg->capacity / 2; // load factor <= 0.5
	return T;
}

static int agg_grow(b200_agg *agg, uint64_t min_capacity) {
	uint64_t new_cap = agg->capacity;
	while (new_cap < min_capacity) {
		new_cap <<= 1;
	}
	if (new_cap == agg->capacity) {
		new_cap <<= 1;
	}
	uint64_t *new_slots = nullptr;
	B200_TRY(agg_alloc_table(agg, new_cap, &new_slots));
	uint64_t *old_slots = agg->slots;
	uint64_t old_cap = agg->capacity;
	agg->slots = new_slots;
	agg->capacity = new_cap;
	AggTable T = agg_table(agg);
	int grid = grid_for(old_cap, 256, 4, agg->ctx->sm_count * 8);
	agg_rehash_kernel<<<grid, 256, 0, agg->ctx->stream>>>(old_slots, old_cap, T, agg->L);
	agg->ctx->launches++;
	b200_dev_free(agg->ctx, old_slots);
	return B200_OK;
}

extern "C" {

int b200_agg_create(b200_ctx *ctx, const int32_t *key_types, int nkeys, const b200_agg_desc *aggs, int naggs,
                    uint64_t expected_groups, b200_agg **out) {
	if (!ctx || !out || nkeys < 1 || nkeys > MAX_KEYS || !key_types || naggs < 0 || naggs > MAX_AGGS ||
	    (naggs > 0 && !aggs)) {
		b200_set_error("b200_agg_create: bad arguments (1..%d keys, 0..%d aggregates)", MAX_KEYS, MAX_AGGS);
		return B200_ERR_INVALID;
	}
	AggLayout L;
	memset(&L, 0, sizeof(L));
	L.nkeys = nkeys;
	int off = 0;
	for (int j = 0; j < nkeys; j++) {
		int sz = b200_type_size(key_types[j]);
		if (!sz || key_types[j] == B200_INT128) {
			b200_set_error("b200_agg_create: unsupported key type %d", key_types[j]);
			return B200_ERR_INVALID;
		}
		if ((off & 7) + sz > 8) {
			off = (off + 7) & ~7;
		}
		L.key_type[j] = key_types[j];
		L.key_off[j] = off;
		off += sz;
	}
	L.null_off = off; // one byte of NULL flags (nkeys <= 8); a single byte never straddles
	off += 1;
	L.key_bytes = off;
	L.key_words = (off + 7) / 8;
	if (L.key_words > KEY_WORDS_MAX) {
		b200_set_error("b200_agg_create: packed group key of %d bytes exceeds %d", off, KEY_WORDS_MAX * 8);
		return B200_ERR_INVALID;
	}
	L.naggs = naggs;
	L.ninputs = 0;
	bool need_sum[MAX_INPUTS] = {false}, need_min[MAX_INPUTS] = {false}, need_max[MAX_INPUTS] = {false};
	for (int a = 0; a < naggs; a++) {
		int f = aggs[a].func, t = aggs[a].input_type, in = aggs[a].input;
		if (f < B200_AGG_COUNT_STAR || f > B200_AGG_AVG) {
			b200_set_error("b200_agg_create: unknown aggregate function %d", f);
			return B200_ERR_INVALID;
		}
		L.func[a] = f;
		if (f == B200_AGG_COUNT_STAR) {
			L.in_type[a] = B200_INT64;
			L.input[a] = -1;
			continue;
		}
		if (!b200_type_size(t) || t == B200_INT128) {
			b200_set_error("b200_agg_create: unsupported aggregate input type %d", t);
			return B200_ERR_INVALID;
		}
		if (f == B200_AGG_SUM_NO_OVERFLOW && !b200_type_is_integer(t)) {
			b200_set_error("b200_agg_create: sum_no_overflow needs an integer input");
			return B200_ERR_INVALID;
		}
		if (in < 0 || in >= MAX_INPUTS) {
			b200_set_error("b200_agg_create: aggregate %d: input index %d out of range [0,%d)", a, in, MAX_INPUTS);
			return B200_ERR_INVALID;
		}
		if (L.input_type[in] && L.input_type[in] != t) {
			b200_set_error("b200_agg_create: aggregates sharing input %d disagree on its type (%d vs %d)", in,
			               L.input_type[in], t);
			return B200_ERR_INVALID;
		}
		L.input_type[in] = t;
		if (in + 1 > L.ninputs) {
			L.ninputs = in + 1;
		}
		L.in_type[a] = t;
		L.input[a] = in;
		need_sum[in] = need_sum[in] || f == B200_AGG_SUM || f == B200_AGG_AVG || f == B200_AGG_SUM_NO_OVERFLOW;
		need_min[in] = need_min[in] || f == B200_AGG_MIN;
		need_max[in] = need_max[in] || f == B200_AGG_MAX;
	}
	for (int i = 0; i < L.ninputs; i++) {
		if (!L.input_type[i]) {
			b200_set_error("b200_agg_create: input %d is not used by any aggregate (inputs must be dense)", i);
			return B200_ERR_INVALID;
		}
	}
	int w = 1 + L.key_words;
	L.rows_off = w++;
	for (int i = 0; i < L.ninputs; i++) {
		L.cnt_off[i] = w++;
		L.sum_off[i] = L.min_off[i] = L.max_off[i] = -1;
		if (need_sum[i]) {
			L.sum_off[i] = w;
			w += b200_type_is_float(L.input_type[i]) ? 1 : 2;
		}
		if (need_min[i]) {
			L.min_off[i] = w++;
		}
		if (need_max[i]) {
			L.max_off[i] = w++;
		}
	}
	L.hash_off = w++; // the full 64-bit hash (used when the table grows)
	L.stride = (w + 3) & ~3;
	b200_agg *agg = new b200_agg();
	memset((void *)agg, 0, sizeof(*agg));
	agg->ctx = ctx;
	agg->L = L;
	cudaSetDevice(ctx->device);
	uint64_t cap = next_pow2(expected_groups ? expected_groups * 2 + 16 : 1 << 16);
	if (cap < (1 << 16)) {
		cap = 1 << 16; // also leaves room for the shared-memory paths' end-of-CTA flushes (they bypass the fill limit)
	}
	agg->capacity = cap;
	int r = agg_alloc_table(agg, cap, &agg->slots);
	void *p = nullptr;
	r = r ? r : b200_dev_alloc(ctx, 8 * 8, &p);
	if (r != B200_OK) {
		b200_agg_destroy(agg);
		return r;
	}
	agg->count = (unsigned long long *)p;
	agg->counters = agg->count + 1;
	cudaMemsetAsync(p, 0, 64, ctx->stream);
	// start optimistic: FAST unless the caller already knows the cardinality is high
	int priv_cap = b200_agg_priv_capacity(L);
	agg->path = expected_groups == 0 || expected_groups <= 4
	                ? PATH_FAST4
	                : (expected_groups <= 8
	                       ? PATH_FAST
	                       : ((int64_t)expected_groups <= priv_cap
	                              ? PATH_PRIV
	                              : (expected_groups <= 2048 ? PATH_MID
	                                                         : (b200_agg_hc_eligible(L) == B200_OK ? PATH_HC : PATH_GLOBAL))));
	agg->path_groups = (int)(expected_groups < 1024 ? expected_groups : 1024);
	agg->path_groups_hc = expected_groups;
	agg->path_decided = false;
	*out = agg;
	return B200_OK;
}

void b200_agg_destroy(b200_agg *agg) {
	if (!agg) {
		return;
	}
	cudaSetDevice(agg->ctx->device);
	b200_agg_hc_destroy(agg->ctx, agg->hc);
	b200_dev_free(agg->ctx, agg->priv_direct_dev);
	b200_dev_free(agg->ctx, agg->slots);
	b200_dev_free(agg->ctx, agg->count);
	delete agg;
}

} // extern "C"

static int read_counters(b200_agg *agg, uint64_t *groups, uint64_t *deferred, uint64_t *missed) {
	b200_ctx *ctx = agg->ctx;
	CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 16, agg->count, 5 * 8, cudaMemcpyDeviceToHost, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	CUDA_TRY(cudaGetLastError());
	ctx->d2h_bytes += 40;
	if (ctx->pinned_scratch[20] & 1) {
		// set by agg_combine_packed_kernel: a source rank held more groups than the packed buffer's max_groups
		b200_set_error("aggregate: a packed partial-state buffer overflowed (more groups than max_groups); use "
		               "b200_agg_export_states / the radix shuffle for this cardinality");
		return B200_ERR_CAPACITY;
	}
	if (groups) {
		*groups = ctx->pinned_scratch[16];
	}
	if (deferred) {
		*deferred = ctx->pinned_scratch[17];
	}
	if (missed) {
		*missed = ctx->pinned_scratch[18];
	}
	return B200_OK;
}

// Run `launch(rows, begin, end, deferred, first)` until no row is deferred, growing the table in between.
// First pass: rows == nullptr, range [begin0, end0).  Later passes: rows = deferred list, range [0, ndef).
static int agg_grow(b200_agg *agg, uint64_t min_capacity);

template <class LAUNCH>
static int run_with_growth(b200_agg *agg, uint64_t begin0, uint64_t end0, LAUNCH launch, uint64_t *missed_out);

template <class LAUNCH, class GROW>
static int run_with_growth(b200_agg *agg, uint64_t begin0, uint64_t end0, LAUNCH launch, uint64_t *missed_out, GROW grow) {
	b200_ctx *ctx = agg->ctx;
	uint32_t *deferred[2] = {nullptr, nullptr};
	uint64_t n = end0 - begin0;
	const uint32_t *rows = nullptr;
	uint64_t b = begin0, e = end0;
	int cur = 0;
	int rc = b200_dev_alloc(ctx, (n + 1) * 4, (void **)&deferred[0]);
	bool first = true;
	while (rc == B200_OK) {
		cudaMemsetAsync(agg->counters, 0, 16, ctx->stream);
		rc = launch(rows, b, e, deferred[cur], first);
		if (rc != B200_OK) {
			break;
		}
		uint64_t ndef = 0, missed = 0;
		rc = read_counters(agg, nullptr, &ndef, &missed);
		if (rc != B200_OK) {
			break;
		}
		if (first && missed_out) {
			*missed_out = missed;
		}
		first = false;
		if (ndef == 0) {
			break;
		}
		rc = grow();
		if (rc != B200_OK) {
			break;
		}
		if (!deferred[1 - cur]) {
			rc = b200_dev_alloc(ctx, (ndef + 1) * 4, (void **)&deferred[1 - cur]);
			if (rc != B200_OK) {
				break;
			}
		}
		rows = deferred[cur];
		b = 0;
		e = ndef;
		cur = 1 - cur;
	}
	b200_dev_free(ctx, deferred[0]);
	b200_dev_free(ctx, deferred[1]);
	return rc;
}

template <class LAUNCH>
static int run_with_growth(b200_agg *agg, uint64_t begin0, uint64_t end0, LAUNCH launch, uint64_t *missed_out) {
	return run_with_growth(agg, begin0, end0, launch, missed_out, [agg]() { return agg_grow(agg, agg->capacity * 4); });
}

// Merge the high-cardinality front-end table into the generic table (before any read-out / combine).
static int read_counters(b200_agg *agg, uint64_t *groups, uint64_t *deferred, uint64_t *missed);
static AggTable agg_table(b200_agg *agg);
static int agg_flush_hc(b200_agg *agg) {
	if (!agg->hc) {
		return B200_OK;
	}
	b200_ctx *ctx = agg->ctx;
	uint64_t hg = 0, groups = 0;
	B200_TRY(b200_agg_hc_groups(ctx, agg->hc, &hg));
	B200_TRY(read_counters(agg, &groups, nullptr, nullptr));
	uint64_t need = 2 * (groups + hg) + 16;
	if (agg->capacity < need) {
		B200_TRY(agg_grow(agg, need));
	}
	AggCols ac;
	memset(&ac, 0, sizeof(ac));
	for (int i = 0; i < agg->L.ninputs; i++) {
		ac.track_cnt[i] = agg->track_cnt[i];
	}
	int rc = b200_agg_hc_flush(ctx, agg->hc, agg->L, agg_table(agg), ac);
	b200_agg_hc_destroy(ctx, agg->hc);
	agg->hc = nullptr;
	agg->aos_empty = false;
	return rc;
}

// PRIV path chosen after the adaptation probe: build the direct addressing tables from the groups found so far
static int agg_build_priv_direct(b200_agg *agg, uint64_t groups, int max_slots) {
	b200_ctx *ctx = agg->ctx;
	agg->priv_direct.nslots = 0;
	const unsigned int MAXG = 1024;
	if (groups == 0 || groups > MAXG || agg->L.key_bytes > 7) {
		return B200_OK;
	}
	uint64_t *list = nullptr;
	B200_TRY(b200_dev_alloc(ctx, MAXG * 8 + 16, (void **)&list));
	unsigned int *counter = (unsigned int *)(list + MAXG);
	cudaMemsetAsync(counter, 0, 8, ctx->stream);
	int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
	agg_list_keys_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, agg->L.stride, list, MAXG, counter);
	ctx->launches++;
	std::vector<uint64_t> host(MAXG + 1);
	cudaError_t e = cudaMemcpyAsync(host.data(), list, (MAXG + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream);
	e = e ? e : cudaStreamSynchronize(ctx->stream);
	b200_dev_free(ctx, list);
	if (e != cudaSuccess) {
		return b200_cuda_fail(e, "agg_build_priv_direct", __FILE__, __LINE__);
	}
	ctx->d2h_bytes += (MAXG + 1) * 8;
	unsigned int n = (unsigned int)(host[MAXG] & 0xffffffffu);
	if (n == 0 || n > MAXG) {
		return B200_OK;
	}
	PrivDirect PD;
	std::vector<uint8_t> tables;
	if (!b200_agg_priv_build_direct(agg->L, host.data(), (int)n, max_slots, &PD, &tables)) {
		return B200_OK;
	}
	b200_dev_free(ctx, agg->priv_direct_dev);
	agg->priv_direct_dev = nullptr;
	B200_TRY(b200_dev_alloc(ctx, tables.size() + 16, &agg->priv_direct_dev));
	e = cudaMemcpyAsync(agg->priv_direct_dev, tables.data(), tables.size(), cudaMemcpyHostToDevice, ctx->stream);
	e = e ? e : cudaStreamSynchronize(ctx->stream); // `tables` is pageable host memory owned by this frame
	if (e != cudaSuccess) {
		return b200_cuda_fail(e, "agg_build_priv_direct(upload)", __FILE__, __LINE__);
	}
	ctx->h2d_bytes += tables.size();
	PD.lut = (const uint8_t *)agg->priv_direct_dev;
	PD.slot_keys = (const unsigned long long *)((const uint8_t *)agg->priv_direct_dev + PD.lut_bytes);
	agg->priv_direct = PD;
	return B200_OK;
}

extern "C" {

int b200_agg_sink(b200_agg *agg, const b200_batch *in, const int *key_cols, const int *input_cols) {
	if (!agg || !in || !key_cols || (agg->L.ninputs > 0 && !input_cols)) {
		b200_set_error("b200_agg_sink: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, L.nkeys, &keys, "b200_agg_sink"));
	for (int j = 0; j < L.nkeys; j++) {
		if (keys.c[j].type != L.key_type[j]) {
			b200_set_error("b200_agg_sink: key %d has type %d, aggregate was created with %d", j, keys.c[j].type,
			               L.key_type[j]);
			return B200_ERR_INVALID;
		}
	}
	AggCols ac;
	memset(&ac, 0, sizeof(ac));
	for (int i = 0; i < L.ninputs; i++) {
		if (input_cols[i] < 0 || input_cols[i] >= (int)in->cols.size()) {
			b200_set_error("b200_agg_sink: aggregate input %d: column %d out of range", i, input_cols[i]);
			return B200_ERR_INVALID;
		}
		ac.c[i] = in->cols[input_cols[i]];
		if (ac.c[i].type != L.input_type[i]) {
			b200_set_error("b200_agg_sink: aggregate input %d has type %d, expected %d", i, ac.c[i].type,
			               L.input_type[i]);
			return B200_ERR_INVALID;
		}
	}
	uint64_t n = in->nrows;
	if (n == 0) {
		return B200_OK;
	}
	if (n > 0xffffffffULL) {
		b200_set_error("b200_agg_sink: at most 2^32-1 rows per batch");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	// inputs that arrive with a validity mask for the first time: start tracking cnt(x)
	for (int i = 0; i < L.ninputs; i++) {
		if (ac.c[i].validity && !agg->track_cnt[i]) {
			if (agg->rows_seen) {
				int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
				agg_fix_cnt_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, i);
				ctx->launches++;
			}
			agg->track_cnt[i] = true;
		}
		ac.track_cnt[i] = agg->track_cnt[i];
	}
	agg->rows_seen += n;
	bool tile_ok = agg->path != PATH_GLOBAL && b200_agg_tile_eligible(L, keys, ac) == B200_OK;
	const bool hc_ok = b200_agg_hc_eligible(L) == B200_OK && !getenv("B200_AGG_NO_HC");
	uint64_t begin = 0;
	while (begin < n) {
		int path = tile_ok ? agg->path : (agg->path == PATH_HC && hc_ok ? PATH_HC : PATH_GLOBAL);
		if ((path == PATH_FAST || path == PATH_FAST4 || path == PATH_PRIV) && L.key_bytes > 7) {
			path = PATH_MID; // FAST / PRIV keep a directory of single-word keys
		}
		if (path == PATH_MID && L.key_words > 2) {
			path = hc_ok ? PATH_HC : PATH_GLOBAL; // the shared-memory table holds two key words
		}
		if (path == PATH_HC && !hc_ok) {
			path = PATH_GLOBAL;
		}
		if (path == PATH_HC) {
			// High cardinality: the L2-first table of agg_hc.cu.  Chunks of 1 M, 2 M, ... 16 M rows; a chunk whose rows
			// find the table at its fill limit defers them, the table doubles and they are replayed; between chunks the
			// table also doubles once it is more than 55 % full.  (Doubling, never more: the table should stay inside
			// L2 for as long as the data allows.)
			if (agg->hc && !b200_agg_hc_compatible(agg->hc, L, agg->track_cnt)) {
				B200_TRY(agg_flush_hc(agg));
			}
			if (!agg->hc) {
				uint64_t g0 = 0;
				B200_TRY(read_counters(agg, &g0, nullptr, nullptr));
				uint64_t hint = 2 * (uint64_t)agg->path_groups_hc;
				B200_TRY(b200_agg_hc_prepare(ctx, &agg->hc, L, agg->track_cnt, hint > 2 * g0 ? hint : 2 * g0));
				// the groups the generic table already holds (the adaptation probe's rows) move into the new table: from
				// here on every group lives there and finalize reads it directly
				if (g0) {
					B200_TRY(b200_agg_hc_absorb(ctx, agg->hc, L, agg->slots, agg->capacity, agg->track_cnt));
					int grid = grid_for(agg->capacity * L.stride, 256, 4, ctx->sm_count * 8);
					agg_init_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L);
					ctx->launches++;
					CUDA_TRY(cudaMemsetAsync(agg->count, 0, 8, ctx->stream));
				}
				agg->aos_empty = true;
			}
			uint64_t chunk = 1ULL << 20;
			int quiet = 0; // consecutive chunks without a deferral or a growth
			while (begin < n) {
				uint64_t end = begin + chunk < n ? begin + chunk : n;
				uint64_t cap_before = b200_agg_hc_capacity(agg->hc);
				int rc = run_with_growth(
				    agg, begin, end,
				    [&](const uint32_t *rows, uint64_t b, uint64_t e, uint32_t *deferred, bool) -> int {
					    return b200_agg_hc_sink(ctx, agg->hc, L, keys, ac, tile_ok, rows, b, e, deferred, agg->counters);
				    },
				    nullptr, [&]() { return b200_agg_hc_grow(ctx, L, agg->hc, b200_agg_hc_capacity(agg->hc) * 2); });
				if (rc != B200_OK) {
					return rc;
				}
				begin = end;
				if (begin < n) {
					uint64_t hg = 0;
					B200_TRY(b200_agg_hc_groups(ctx, agg->hc, &hg));
					uint64_t cap = b200_agg_hc_capacity(agg->hc);
					if (hg * 20 > cap * 11) {
						B200_TRY(b200_agg_hc_grow(ctx, L, agg->hc, cap * 2));
					}
				}
				quiet = b200_agg_hc_capacity(agg->hc) == cap_before ? quiet + 1 : 0;
				if (chunk < (1ULL << 24)) {
					chunk <<= 1;
				} else if (quiet >= 2) {
					chunk = n; // the table has stopped growing: the rest of the batch in one launch
				}
			}
			b200_agg_hc_unpin(ctx, agg->hc);
			break;
		}
		// while the path is undecided, sink a probe chunk and look at how many groups it holds
		uint64_t end = n;
		if (path != PATH_GLOBAL && !agg->path_decided) {
			end = begin + (1ULL << 18) < n ? begin + (1ULL << 18) : n;
		}
		if (path != PATH_GLOBAL) {
			// the shared-memory paths flush their per-CTA groups at the end of the kernel WITHOUT the fill-limit
			// check: keep 4x that many slots so the flushes always find room (load factor stays <= 0.75)
			uint64_t need = 4 * b200_agg_tile_headroom(path == PATH_MID ? 1 : (path == PATH_PRIV ? 2 : 0), ctx->sm_count);
			if (agg->capacity < need) {
				B200_TRY(agg_grow(agg, need));
			}
		}
		uint64_t missed = 0;
		int rc = run_with_growth(
		    agg, begin, end,
		    [&](const uint32_t *rows, uint64_t b, uint64_t e, uint32_t *deferred, bool first) -> int {
			    if (first && path != PATH_GLOBAL) {
				    return b200_agg_tile_sink(ctx, path == PATH_MID ? 1 : (path == PATH_PRIV ? 2 : 0),
				                              path == PATH_FAST4 ? 4 : (path == PATH_PRIV ? agg->path_groups : 16), L,
				                              agg_table(agg), keys, ac, b, e, deferred, agg->counters,
				                              path == PATH_PRIV ? &agg->priv_direct : nullptr);
			    }
			    int grid = grid_for(e - b, 256, 4, ctx->sm_count * 8);
			    agg_sink_kernel<<<grid, 256, 0, ctx->stream>>>(agg_table(agg), L, keys, ac, b, e, rows, deferred,
			                                                   agg->counters);
			    ctx->launches++;
			    return B200_OK;
		    },
		    &missed);
		if (rc != B200_OK) {
			return rc;
		}
		if (path != PATH_GLOBAL && !agg->path_decided) {
			// adaptation (the analogue of DecideAdaptation's HyperLogLog estimate): every row of the probe chunk has
			// been aggregated - in shared memory or, on a miss, inline in the global table - so the table's group
			// count is the exact cardinality of the first rows.  Pick the cheapest structure that holds it.
			uint64_t groups = 0;
			B200_TRY(read_counters(agg, &groups, nullptr, nullptr));
			const char *priv_env = getenv("B200_AGG_PRIV"); // experiment knob: 0 = never PRIV, 2 = PRIV also for <= 8 groups
			int priv_mode = priv_env ? atoi(priv_env) : 1;
			int priv_cap = priv_mode ? b200_agg_priv_capacity(L) : 0;
			agg->path_groups = (int)(groups < 1024 ? groups : 1024);
			agg->path_groups_hc = groups;
			if (priv_mode == 2 && (int64_t)groups <= priv_cap) {
				agg->path = PATH_PRIV;
			} else if (groups <= 4) {
				agg->path = PATH_FAST4;
			} else if (groups <= 8) {
				agg->path = PATH_FAST;
			} else if ((int64_t)groups <= priv_cap) {
				agg->path = PATH_PRIV;
			} else if (groups <= 700) {
				agg->path = PATH_MID; // (only shapes PRIV / WPRIV do not take get here with <= ~1000 groups)
			} else {
				agg->path = hc_ok ? PATH_HC : PATH_GLOBAL;
			}
			agg->path_decided = true;
			(void)missed;
			if (agg->path == PATH_PRIV) {
				B200_TRY(agg_build_priv_direct(agg, groups, priv_cap));
			}
		}
		begin = end;
	}
	return B200_OK;
}

int b200_agg_group_count(b200_agg *agg, uint64_t *out_groups) {
	if (!agg || !out_groups) {
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(agg->ctx->device));
	if (agg->hc && agg->aos_empty) {
		return b200_agg_hc_groups(agg->ctx, agg->hc, out_groups);
	}
	B200_TRY(agg_flush_hc(agg));
	return read_counters(agg, out_groups, nullptr, nullptr);
}

int b200_agg_finalize(b200_agg *agg, b200_batch **out) {
	if (!agg || !out) {
		b200_set_error("b200_agg_finalize: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	CUDA_TRY(cudaSetDevice(ctx->device));
	const bool from_hc = agg->hc && agg->aos_empty; // every group lives in the high-cardinality table: read it directly
	uint64_t groups = 0;
	if (from_hc) {
		B200_TRY(read_counters(agg, nullptr, nullptr, nullptr)); // (reports a packed-buffer overflow, if any)
		B200_TRY(b200_agg_hc_groups(ctx, agg->hc, &groups));
	} else {
		B200_TRY(agg_flush_hc(agg));
		B200_TRY(read_counters(agg, &groups, nullptr, nullptr));
	}
	b200_batch *ob = b200_batch_new(ctx, groups);
	FinalizeOut fo;
	memset(&fo, 0, sizeof(fo));
	for (int i = 0; i < L.ninputs; i++) {
		fo.track_cnt[i] = agg->track_cnt[i];
	}
	uint64_t words = (groups + 63) / 64;
	int rc = B200_OK;
	for (int j = 0; j < L.nkeys && rc == B200_OK; j++) {
		rc = b200_batch_add_flat(ob, L.key_type[j], groups, true, &fo.key_data[j], &fo.key_valid[j]);
		if (rc == B200_OK && words) {
			fill_u64_kernel3<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(fo.key_valid[j], words, ~0ULL);
			ctx->launches++;
		}
	}
	std::vector<void *> avg_raw(L.naggs, nullptr);
	for (int a = 0; a < L.naggs && rc == B200_OK; a++) {
		int rt = agg_result_type(L.func[a], L.in_type[a]);
		rc = b200_batch_add_flat(ob, rt, groups, true, &fo.agg_data[a], &fo.agg_valid[a]);
		if (rc == B200_OK && words) {
			fill_u64_kernel3<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(fo.agg_valid[a], words, ~0ULL);
			ctx->launches++;
		}
		if (rc == B200_OK && L.func[a] == B200_AGG_AVG && !b200_type_is_float(L.in_type[a])) {
			rc = b200_dev_alloc(ctx, (size_t)groups * 24 + 16, &avg_raw[a]);
			if (rc == B200_OK) {
				std::swap(fo.agg_data[a], avg_raw[a]); // kernel writes raw triples; column filled by the host
			}
		}
	}
	if (rc != B200_OK) {
		b200_batch_free(ob);
		return rc;
	}
	unsigned long long *out_counter = agg->counters + 2;
	cudaMemsetAsync(out_counter, 0, 8, ctx->stream);
	if (groups && from_hc) {
		int hrc = b200_agg_hc_finalize(ctx, agg->hc, L, fo, out_counter);
		if (hrc != B200_OK) {
			b200_batch_free(ob);
			return hrc;
		}
	} else if (groups) {
		int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
		agg_finalize_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, fo, out_counter);
		ctx->launches++;
	}
	// integer AVG: finish on the host in long double, bit-exact with
	// IntegerAverageOperationHugeint::Finalize (avg.cpp:109-121): Hugeint::Cast<long double>(sum) / count
	for (int a = 0; a < L.naggs; a++) {
		if (!avg_raw[a]) {
			continue;
		}
		void *raw_dev = fo.agg_data[a];
		void *col_dev = avg_raw[a];
		std::vector<uint64_t> raw(groups * 3);
		std::vector<double> res(groups);
		if (groups) {
			cudaError_t e = cudaMemcpyAsync(raw.data(), raw_dev, groups * 24, cudaMemcpyDeviceToHost, ctx->stream);
			e = e ? e : cudaStreamSynchronize(ctx->stream);
			if (e != cudaSuccess) {
				for (int q = a; q < L.naggs; q++) {
					if (avg_raw[q]) {
						b200_dev_free(ctx, fo.agg_data[q]); // the raw triples of the averages not finished yet
					}
				}
				b200_batch_free(ob);
				return b200_cuda_fail(e, "avg finalize D2H", __FILE__, __LINE__);
			}
			ctx->d2h_bytes += groups * 24;
			bool is_signed = b200_type_is_signed_int(L.in_type[a]);
			for (uint64_t g = 0; g < groups; g++) {
				uint64_t lo = raw[3 * g], hi = raw[3 * g + 1], cnt = raw[3 * g + 2];
				long double v;
				if (is_signed && (int64_t)hi < 0) {
					// negate the 128-bit value, convert, negate (Hugeint::Cast<long double>)
					uint64_t nlo = ~lo + 1, nhi = ~hi + (nlo == 0 ? 1 : 0);
					v = -((long double)nhi * 18446744073709551616.0L + (long double)nlo);
				} else {
					v = (long double)hi * 18446744073709551616.0L + (long double)lo;
				}
				res[g] = cnt ? (double)(v / (long double)cnt) : 0.0;
			}
			e = cudaMemcpyAsync(col_dev, res.data(), groups * 8, cudaMemcpyHostToDevice, ctx->stream);
			e = e ? e : cudaStreamSynchronize(ctx->stream);
			if (e != cudaSuccess) {
				for (int q = a; q < L.naggs; q++) {
					if (avg_raw[q]) {
						b200_dev_free(ctx, fo.agg_data[q]);
					}
				}
				b200_batch_free(ob);
				return b200_cuda_fail(e, "avg finalize H2D", __FILE__, __LINE__);
			}
			ctx->h2d_bytes += groups * 8;
		}
		b200_dev_free(ctx, raw_dev);
	}
	cudaError_t e = cudaStreamSynchronize(ctx->stream);
	e = e ? e : cudaGetLastError();
	if (e != cudaSuccess) {
		b200_batch_free(ob);
		return b200_cuda_fail(e, "agg_finalize", __FILE__, __LINE__);
	}
	*out = ob;
	return B200_OK;
}

int b200_agg_export_states(b200_agg *agg, b200_batch **out) {
	if (!agg || !out) {
		b200_set_error("b200_agg_export_states: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	CUDA_TRY(cudaSetDevice(ctx->device));
	B200_TRY(agg_flush_hc(agg));
	uint64_t groups = 0;
	B200_TRY(read_counters(agg, &groups, nullptr, nullptr));
	b200_batch *ob = b200_batch_new(ctx, groups);
	ExportOut eo;
	memset(&eo, 0, sizeof(eo));
	for (int i = 0; i < L.ninputs; i++) {
		eo.track_cnt[i] = agg->track_cnt[i];
	}
	StateMap sm;
	state_map(L, &sm);
	uint64_t words = (groups + 63) / 64;
	int rc = B200_OK;
	for (int j = 0; j < L.nkeys && rc == B200_OK; j++) {
		rc = b200_batch_add_flat(ob, L.key_type[j], groups, true, &eo.key_data[j], &eo.key_valid[j]);
		if (rc == B200_OK && words) {
			fill_u64_kernel3<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(eo.key_valid[j], words, ~0ULL);
			ctx->launches++;
		}
	}
	for (int c = 0; c < sm.n && rc == B200_OK; c++) {
		void *d = nullptr;
		rc = b200_batch_add_flat(ob, B200_UINT64, groups, false, &d, nullptr);
		eo.state_cols[c] = (uint64_t *)d;
	}
	if (rc != B200_OK) {
		b200_batch_free(ob);
		return rc;
	}
	unsigned long long *out_counter = agg->counters + 2;
	cudaMemsetAsync(out_counter, 0, 8, ctx->stream);
	if (groups) {
		int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
		agg_export_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, eo, sm, out_counter);
		ctx->launches++;
	}
	cudaError_t e = cudaStreamSynchronize(ctx->stream);
	e = e ? e : cudaGetLastError();
	if (e != cudaSuccess) {
		b200_batch_free(ob);
		return b200_cuda_fail(e, "agg_export_states", __FILE__, __LINE__);
	}
	*out = ob;
	return B200_OK;
}

int b200_agg_combine_states(b200_agg *agg, const b200_batch *states) {
	if (!agg || !states) {
		b200_set_error("b200_agg_combine_states: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	StateMap sm;
	state_map(L, &sm);
	if ((int)states->cols.size() != L.nkeys + sm.n) {
		b200_set_error("b200_agg_combine_states: expected %d columns, got %d", L.nkeys + sm.n,
		               (int)states->cols.size());
		return B200_ERR_INVALID;
	}
	KeyCols keys;
	keys.n = L.nkeys;
	for (int j = 0; j < L.nkeys; j++) {
		keys.c[j] = states->cols[j];
		if (keys.c[j].type != L.key_type[j]) {
			b200_set_error("b200_agg_combine_states: key %d type mismatch", j);
			return B200_ERR_INVALID;
		}
	}
	StateCols sc;
	for (int i = 0; i < sm.n; i++) {
		const DCol &c = states->cols[L.nkeys + i];
		if (c.type != B200_UINT64 || c.vtype != B200_FLAT_VECTOR) {
			b200_set_error("b200_agg_combine_states: state column %d must be a flat UINT64 column", i);
			return B200_ERR_INVALID;
		}
		sc.c[i] = (const uint64_t *)c.data;
	}
	uint64_t n = states->nrows;
	if (n == 0) {
		return B200_OK;
	}
	if (n > 0xffffffffULL) {
		b200_set_error("b200_agg_combine_states: at most 2^32-1 rows per batch");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	B200_TRY(agg_flush_hc(agg));
	// exported states carry an explicit cnt(x) for every input: from now on cnt is tracked here as well
	for (int i = 0; i < L.ninputs; i++) {
		if (!agg->track_cnt[i]) {
			if (agg->rows_seen) {
				int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
				agg_fix_cnt_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, i);
				ctx->launches++;
			}
			agg->track_cnt[i] = true;
		}
	}
	agg->rows_seen += n;
	return run_with_growth(
	    agg, 0, n,
	    [&](const uint32_t *rows, uint64_t b, uint64_t e, uint32_t *deferred, bool) -> int {
		    int grid = grid_for(e - b, 256, 4, ctx->sm_count * 8);
		    agg_combine_kernel<<<grid, 256, 0, ctx->stream>>>(agg_table(agg), L, keys, sc, b, e, rows, deferred,
		                                                      agg->counters);
		    ctx->launches++;
		    return B200_OK;
	    },
	    nullptr);
}

uint64_t b200_agg_packed_words(b200_agg *agg, uint64_t max_groups) {
	if (!agg) {
		return 0;
	}
	StateMap sm;
	state_map(agg->L, &sm);
	return 2 + (uint64_t)(agg->L.nkeys + 1 + sm.n) * max_groups;
}

int b200_agg_export_packed(b200_agg *agg, uint64_t *dst_dev, uint64_t max_groups) {
	if (!agg || !dst_dev || max_groups == 0) {
		b200_set_error("b200_agg_export_packed: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	CUDA_TRY(cudaSetDevice(ctx->device));
	B200_TRY(agg_flush_hc(agg));
	ExportOut eo;
	memset(&eo, 0, sizeof(eo));
	for (int i = 0; i < L.ninputs; i++) {
		eo.track_cnt[i] = agg->track_cnt[i];
	}
	StateMap sm;
	state_map(L, &sm);
	unsigned long long *out_counter = agg->counters + 2;
	CUDA_TRY(cudaMemsetAsync(out_counter, 0, 8, ctx->stream));
	int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
	agg_export_packed_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, sm, eo, dst_dev, max_groups,
	                                                        out_counter);
	agg_packed_header_kernel<<<1, 1, 0, ctx->stream>>>(dst_dev, max_groups, out_counter);
	ctx->launches += 2;
	CUDA_TRY(cudaGetLastError());
	return B200_OK; // stream-asynchronous: no host round trip
}

int b200_agg_combine_packed(b200_agg *agg, const uint64_t *src_dev, int nranks, uint64_t max_groups) {
	if (!agg || !src_dev || nranks < 1 || max_groups == 0) {
		b200_set_error("b200_agg_combine_packed: bad arguments");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = agg->ctx;
	const AggLayout &L = agg->L;
	CUDA_TRY(cudaSetDevice(ctx->device));
	B200_TRY(agg_flush_hc(agg));
	// no deferral on this path: the table must have room for everything already in it plus every incoming group
	uint64_t incoming = (uint64_t)nranks * max_groups;
	if (agg->rows_seen != 0) {
		uint64_t groups = 0;
		B200_TRY(read_counters(agg, &groups, nullptr, nullptr));
		incoming += groups;
	}
	if (agg->capacity < 2 * incoming + 16) {
		B200_TRY(agg_grow(agg, 2 * incoming + 16));
	}
	for (int i = 0; i < L.ninputs; i++) {
		if (!agg->track_cnt[i]) {
			if (agg->rows_seen) {
				int grid = grid_for(agg->capacity, 256, 4, ctx->sm_count * 8);
				agg_fix_cnt_kernel<<<grid, 256, 0, ctx->stream>>>(agg->slots, agg->capacity, L, i);
				ctx->launches++;
			}
			agg->track_cnt[i] = true;
		}
	}
	agg->rows_seen += 1;
	StateMap sm;
	state_map(L, &sm);
	uint64_t words = 2 + (uint64_t)(L.nkeys + 1 + sm.n) * max_groups;
	agg_combine_packed_kernel<<<nranks, 128, 0, ctx->stream>>>(agg_table(agg), L, sm, src_dev, words, nranks, max_groups,
	                                                           agg->counters);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK; // an overflowed source buffer is reported by b200_agg_finalize (B200_ERR_CAPACITY)
}

} // extern "C"
