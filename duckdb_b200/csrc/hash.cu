// K1 hash_keys and K2 radix_partition.
// Reference semantics: VectorOperations::Hash / CombineHash
// (src/common/vector_operations/vector_hash.cpp:24-49,504-552), duckdb::Hash<T>
// (src/include/duckdb/common/types/hash.hpp:38-54), RadixPartitioning::ApplyMask
// (src/include/duckdb/common/radix_partitioning.hpp:45-61).
#include "common.cuh"
#include <utility>
#include <cstdlib>

int b200_fill_keycols(const b200_batch *b, const int *cols, int n, KeyCols *out, const char *who) {
	if (n < 1 || n > MAX_KEYS) {
		b200_set_error("%s: between 1 and %d key columns are supported (got %d)", who, MAX_KEYS, n);
		return B200_ERR_INVALID;
	}
	out->n = n;
	for (int j = 0; j < n; j++) {
		if (cols[j] < 0 || cols[j] >= (int)b->cols.size()) {
			b200_set_error("%s: key column index %d out of range", who, cols[j]);
			return B200_ERR_INVALID;
		}
		out->c[j] = b->cols[cols[j]];
		if (out->c[j].type == B200_INT128) {
			b200_set_error("%s: INT128 keys are not supported", who);
			return B200_ERR_INVALID;
		}
	}
	return B200_OK;
}

__global__ void __launch_bounds__(256) hash_kernel(KeyCols keys, uint64_t n, uint64_t *__restrict__ out) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		bool nul;
		out[row] = hash_row(keys, row, &nul);
	}
}

// ---------------------------------------------------------------- radix partition
// Pass 1: per-block histogram in shared memory -> global counts (one atomic per block per bucket).
// Pass 2: each block claims, per bucket, a contiguous range with one global atomicAdd, then scatters.
#define PART_MAX 4096
#define TP_MAX_PART_COLS 16

__global__ void __launch_bounds__(256)
    part_hist_kernel(KeyCols keys, uint64_t n, int bits, unsigned long long *__restrict__ counts,
                     uint32_t *__restrict__ part_of_row) {
	extern __shared__ uint32_t sh[];
	int nparts = 1 << bits;
	for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
		sh[i] = 0;
	}
	__syncthreads();
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		bool nul;
		uint64_t h = hash_row(keys, row, &nul);
		uint32_t p = (uint32_t)((h >> (48 - bits)) & (uint64_t)(nparts - 1));
		part_of_row[row] = p;
		atomicAdd(&sh[p], 1u);
	}
	__syncthreads();
	for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
		if (sh[i]) {
			atomicAdd(&counts[i], (unsigned long long)sh[i]);
		}
	}
}

// tile = blockDim.x * ROWS rows per block iteration; order inside a partition is unspecified
__global__ void __launch_bounds__(256)
    part_scatter_index_kernel(const uint32_t *__restrict__ part_of_row, uint64_t n, int bits,
                              unsigned long long *__restrict__ cursors, uint32_t *__restrict__ dest_of_row) {
	extern __shared__ uint32_t sh[]; // [nparts] counts, then [nparts*2] base (as 64-bit)
	int nparts = 1 << bits;
	uint32_t *cnt = sh;
	unsigned long long *base = (unsigned long long *)(sh + nparts + (nparts & 1));
	const int ROWS = 8;
	uint64_t tile = (uint64_t)blockDim.x * ROWS;
	for (uint64_t start = (uint64_t)blockIdx.x * tile; start < n; start += (uint64_t)gridDim.x * tile) {
		for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
			cnt[i] = 0;
		}
		__syncthreads();
		uint32_t p[ROWS], r[ROWS];
#pragma unroll
		for (int k = 0; k < ROWS; k++) {
			uint64_t row = start + (uint64_t)k * blockDim.x + threadIdx.x;
			if (row < n) {
				p[k] = part_of_row[row];
				r[k] = atomicAdd(&cnt[p[k]], 1u);
			}
		}
		__syncthreads();
		for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
			base[i] = cnt[i] ? atomicAdd(&cursors[i], (unsigned long long)cnt[i]) : 0ULL;
		}
		__syncthreads();
#pragma unroll
		for (int k = 0; k < ROWS; k++) {
			uint64_t row = start + (uint64_t)k * blockDim.x + threadIdx.x;
			if (row < n) {
				dest_of_row[row] = (uint32_t)(base[p[k]] + r[k]);
			}
		}
		__syncthreads();
	}
}

// scatter one column to its destination slots (flattening const/dict inputs)
__global__ void __launch_bounds__(256)
    part_scatter_col_kernel(DCol c, uint64_t n, const uint32_t *__restrict__ dest_of_row, void *__restrict__ out,
                            uint64_t *__restrict__ out_validity) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		uint64_t idx = col_index(c, row);
		uint32_t d = dest_of_row[row];
		store_raw(out, c.type, d, col_load_raw(c, idx));
		if (out_validity && !col_valid_at(c, idx)) {
			atomicAnd((unsigned long long *)&out_validity[d >> 6], ~(1ULL << (d & 63)));
		}
	}
}

__global__ void fill_u64_kernel(uint64_t *p, uint64_t words, uint64_t v) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) {
		p[i] = v;
	}
}

__global__ void exclusive_scan_small_kernel(const unsigned long long *counts, unsigned long long *cursors, int n) {
	if (threadIdx.x == 0 && blockIdx.x == 0) {
		unsigned long long acc = 0;
		for (int i = 0; i < n; i++) {
			cursors[i] = acc;
			acc += counts[i];
		}
	}
}

// ---------------------------------------------------------------- radix partition, fast path (<= 16 partitions)
// Two passes, no per-row scratch arrays:
//   1. part_count_kernel         partition id from the key hash; the lanes of a warp that share a partition find each
//                                other with ONE match.any (SASS MATCH.ANY) and their leader adds the group's size to
//                                a per-CTA counter: one shared-memory atomic per (warp instruction, distinct
//                                partition), one global atomic per (CTA, partition)
//   2. part_move_staged_kernel   recompute the id, rank the row inside its (tile, partition) the same way, order the
//                                2048-row tile by partition in SHARED memory, claim ONE global range per (tile,
//                                partition) and copy every partition's run out with consecutive threads on consecutive
//                                addresses: stores are coalesced whatever the partition count, and the runs are what
//                                a peer-memory (NVLink) destination needs.
// Eligibility: bits <= 4, all columns FLAT without validity, a 2048-row tile of all columns fits 96 KB.
// (One ballot per partition per row - 16 unrolled ballots - makes the kernel issue-bound; match.any replaces them.)
#define PF_MAXP 16
#define PF_THREADS 256
#define PF_ROWS 8

struct PartCols {
	const void *in[TP_MAX_PART_COLS];
	void *out[TP_MAX_PART_COLS];
	int width[TP_MAX_PART_COLS];
	int n;
};

// partition of `row`; FAST64: one flat 8-byte integer key without NULLs (TPC-H keys are BIGINT)
template <bool FAST64>
__device__ __forceinline__ uint32_t part_of(const KeyCols &keys, uint64_t row, int bits) {
	uint64_t h;
	if (FAST64) {
		h = murmur64(__ldg((const uint64_t *)keys.c[0].data + row));
	} else {
		bool nul;
		h = hash_row(keys, row, &nul);
	}
	return (uint32_t)((h >> (48 - bits)) & (uint64_t)((1u << bits) - 1));
}

static bool keys_fast64(const KeyCols &keys) {
	return keys.n == 1 && (keys.c[0].type == B200_INT64 || keys.c[0].type == B200_UINT64) &&
	       keys.c[0].vtype == B200_FLAT_VECTOR && !keys.c[0].validity;
}

template <bool FAST64>
__global__ void __launch_bounds__(PF_THREADS)
    part_count_kernel(KeyCols keys, uint64_t n, int bits, unsigned long long *__restrict__ counts) {
	__shared__ unsigned int sh[PF_MAXP];
	const int lane = threadIdx.x & 31;
	if (threadIdx.x < PF_MAXP) {
		sh[threadIdx.x] = 0;
	}
	__syncthreads();
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	uint64_t n_round = (n + 31) / 32 * 32;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_round; row += stride) {
		uint32_t my = row < n ? part_of<FAST64>(keys, row, bits) : 0xffffffffu;
		uint32_t m = __match_any_sync(0xffffffffu, my);
		if (my != 0xffffffffu && lane == __ffs(m) - 1) {
			atomicAdd(&sh[my], (unsigned int)__popc(m));
		}
	}
	__syncthreads();
	if (threadIdx.x < (1 << bits) && sh[threadIdx.x]) {
		atomicAdd(&counts[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
	}
}

// PEER = true: partition p's run goes to dst.out[p][c] (a buffer on GPU p, mapped through NVLink peer memory) instead of
// the one local output batch - the partition scatter and the transfer are ONE kernel (b200_partition_scatter).
struct PartDst {
	void *out[PF_MAXP][TP_MAX_PART_COLS];
};

template <bool PEER, bool FAST64>
__global__ void __launch_bounds__(PF_THREADS)
    part_move_staged_kernel(KeyCols keys, PartCols pc, const __grid_constant__ PartDst dst, uint64_t n, int bits,
                            unsigned long long *__restrict__ cursors, uint64_t capacity, unsigned long long *dropped) {
	extern __shared__ __align__(16) unsigned char stage_raw[]; // column c of the tile (TILE values each), then ppart[TILE]
	constexpr uint32_t TILE = PF_THREADS * PF_ROWS;
	__shared__ unsigned int tcnt[PF_MAXP];       // rows of the tile per partition (atomic ranks)
	__shared__ unsigned int pstart[PF_MAXP + 1];  // start of the partition's run inside the staged tile
	__shared__ unsigned long long base[PF_MAXP]; // claimed global start of the partition's run
	const int nparts = 1 << bits, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t col_off[TP_MAX_PART_COLS];
	uint32_t off = 0;
	for (int c = 0; c < pc.n; c++) {
		col_off[c] = off;
		off += (uint32_t)pc.width[c] * TILE; // widths are 1/2/4/8 and TILE is a multiple of 8: offsets stay aligned
	}
	uint8_t *ppart = stage_raw + off; // partition of every staged position
	for (uint64_t start = (uint64_t)blockIdx.x * TILE; start < n; start += (uint64_t)gridDim.x * TILE) {
		const uint32_t rows_in_tile = n - start < TILE ? (uint32_t)(n - start) : TILE;
		if (threadIdx.x < PF_MAXP) {
			tcnt[threadIdx.x] = 0;
		}
		__syncthreads();
		uint32_t part[PF_ROWS], rank[PF_ROWS];
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			uint64_t row = start + (uint64_t)k * PF_THREADS + threadIdx.x;
			part[k] = row < n ? part_of<FAST64>(keys, row, bits) : 0xffffffffu;
			// the lanes of this warp instruction that go to the same partition: one MATCH, the leader claims their ranks
			uint32_t m = __match_any_sync(0xffffffffu, part[k]);
			int leader = __ffs(m) - 1;
			uint32_t b = 0;
			if (lane == leader && part[k] != 0xffffffffu) {
				b = atomicAdd(&tcnt[part[k]], (unsigned int)__popc(m));
			}
			rank[k] = __shfl_sync(0xffffffffu, b, leader) + __popc(m & ((1u << lane) - 1));
		}
		__syncthreads();
		if (warp == 0) {
			// exclusive prefix of the <= 16 partition counts; claim the global ranges
			uint32_t c = lane < nparts ? tcnt[lane] : 0, incl = c;
#pragma unroll
			for (int d = 1; d < PF_MAXP; d <<= 1) {
				uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
				if (lane >= d) {
					incl += t;
				}
			}
			if (lane < nparts) {
				pstart[lane] = incl - c;
				base[lane] = c ? atomicAdd(&cursors[lane], (unsigned long long)c) : 0ULL;
			}
			if (lane == nparts - 1) {
				pstart[nparts] = incl;
			}
		}
		__syncthreads();
		// local scatter: the thread's rows go to their partition-ordered position in shared memory
		uint32_t lpos[PF_ROWS];
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			lpos[k] = part[k] == 0xffffffffu ? 0 : pstart[part[k]] + rank[k];
			if (part[k] != 0xffffffffu) {
				ppart[lpos[k]] = (uint8_t)part[k];
			}
		}
#pragma unroll 1
		for (int c = 0; c < pc.n; c++) {
			unsigned char *sc = stage_raw + col_off[c];
			switch (pc.width[c]) {
			case 1:
#pragma unroll
				for (int k = 0; k < PF_ROWS; k++) {
					if (part[k] != 0xffffffffu) {
						((uint8_t *)sc)[lpos[k]] = ((const uint8_t *)pc.in[c])[start + (uint64_t)k * PF_THREADS + threadIdx.x];
					}
				}
				break;
			case 2:
#pragma unroll
				for (int k = 0; k < PF_ROWS; k++) {
					if (part[k] != 0xffffffffu) {
						((uint16_t *)sc)[lpos[k]] = ((const uint16_t *)pc.in[c])[start + (uint64_t)k * PF_THREADS + threadIdx.x];
					}
				}
				break;
			case 4:
#pragma unroll
				for (int k = 0; k < PF_ROWS; k++) {
					if (part[k] != 0xffffffffu) {
						((uint32_t *)sc)[lpos[k]] = ((const uint32_t *)pc.in[c])[start + (uint64_t)k * PF_THREADS + threadIdx.x];
					}
				}
				break;
			default:
#pragma unroll
				for (int k = 0; k < PF_ROWS; k++) {
					if (part[k] != 0xffffffffu) {
						((uint64_t *)sc)[lpos[k]] = ((const uint64_t *)pc.in[c])[start + (uint64_t)k * PF_THREADS + threadIdx.x];
					}
				}
				break;
			}
		}
		__syncthreads();
		// copy out: consecutive threads hold consecutive positions of the same run -> consecutive global addresses
		uint64_t pos[PF_ROWS];
		uint32_t pp[PF_ROWS];
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			uint32_t i = k * PF_THREADS + threadIdx.x;
			pp[k] = i < rows_in_tile ? ppart[i] : 0xffffffffu;
			pos[k] = i < rows_in_tile ? base[pp[k]] + (i - pstart[pp[k]]) : 0;
			if (PEER && pp[k] != 0xffffffffu && pos[k] >= capacity) {
				// a receive buffer too small for this exchange: never write past it; the host reads the count and raises
				atomicAdd(dropped, 1ULL);
				pp[k] = 0xffffffffu;
			}
		}
#pragma unroll 1
		for (int c = 0; c < pc.n; c++) {
			const unsigned char *sc = stage_raw + col_off[c];
#pragma unroll
			for (int k = 0; k < PF_ROWS; k++) {
				if (pp[k] == 0xffffffffu) {
					continue;
				}
				uint32_t i = k * PF_THREADS + threadIdx.x;
				void *out = PEER ? dst.out[pp[k]][c] : pc.out[c];
				switch (pc.width[c]) {
				case 1:
					((uint8_t *)out)[pos[k]] = ((const uint8_t *)sc)[i];
					break;
				case 2:
					((uint16_t *)out)[pos[k]] = ((const uint16_t *)sc)[i];
					break;
				case 4:
					((uint32_t *)out)[pos[k]] = ((const uint32_t *)sc)[i];
					break;
				default:
					((uint64_t *)out)[pos[k]] = ((const uint64_t *)sc)[i];
					break;
				}
			}
		}
		__syncthreads(); // tcnt / pstart / base / the stage are rewritten by the next tile
	}
}

// The same kernel for the shape the shuffle-join moves (NC 8-byte columns, the BIGINT key among them, column 0 here):
// ALL global loads of a tile are issued up front into registers (8 rows x NC values per thread), the key is hashed from
// its register copy instead of being read twice, and the loads complete behind the match / rank / prefix phases.
// (A shared-memory store that waits for the load right in front of it makes the kernel latency-bound.)
// BULK: every (partition, column) run of the staged tile leaves with ONE bulk-async copy (cp.async.bulk shared -> global,
// SASS UBLKCP) instead of 8-byte stores - a few large NVLink writes per tile instead of thousands of small ones.  Runs
// are padded in shared memory so that source and destination share their 16-byte phase; an odd head / tail element
// goes by a plain store.
#define PF_PAD 32
__device__ __forceinline__ void pf_bulk_store(void *gdst, const void *ssrc, uint32_t bytes) {
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
	             "r"((uint32_t)__cvta_generic_to_shared(ssrc)), "r"(bytes)
	             : "memory");
}

template <bool PEER, int NC, bool BULK>
__global__ void __launch_bounds__(PF_THREADS, 2)
    part_move_reg_kernel(PartCols pc, const __grid_constant__ PartDst dst, uint64_t n, int bits,
                         unsigned long long *__restrict__ cursors, uint64_t capacity, unsigned long long *dropped) {
	extern __shared__ __align__(16) unsigned char stage_raw[]; // NC columns of CS 8-byte values (, then ppart[TILE])
	constexpr uint32_t TILE = PF_THREADS * PF_ROWS;
	constexpr uint32_t CS = BULK ? TILE + PF_PAD : TILE; // column stride in values
	__shared__ unsigned int tcnt[PF_MAXP];
	__shared__ unsigned int pstart[PF_MAXP + 1];
	__shared__ unsigned long long base[PF_MAXP];
	const int nparts = 1 << bits, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint64_t *stage = (uint64_t *)stage_raw;
	uint8_t *ppart = stage_raw + (size_t)NC * CS * 8;
	const uint64_t pmask = (uint64_t)((1u << bits) - 1);
	for (uint64_t start = (uint64_t)blockIdx.x * TILE; start < n; start += (uint64_t)gridDim.x * TILE) {
		const uint32_t rows_in_tile = n - start < TILE ? (uint32_t)(n - start) : TILE;
		if (threadIdx.x < PF_MAXP) {
			tcnt[threadIdx.x] = 0;
		}
		// every load of the tile, back to back
		uint64_t v[PF_ROWS][NC];
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			const uint32_t i = k * PF_THREADS + threadIdx.x;
#pragma unroll
			for (int c = 0; c < NC; c++) {
				v[k][c] = i < rows_in_tile ? __ldcs((const unsigned long long *)pc.in[c] + start + i) : 0ULL;
			}
		}
		__syncthreads();
		uint32_t part[PF_ROWS], rank[PF_ROWS];
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			const uint32_t i = k * PF_THREADS + threadIdx.x;
			part[k] = i < rows_in_tile ? (uint32_t)((murmur64(v[k][0]) >> (48 - bits)) & pmask) : 0xffffffffu;
			uint32_t m = __match_any_sync(0xffffffffu, part[k]);
			int leader = __ffs(m) - 1;
			uint32_t b = 0;
			if (lane == leader && part[k] != 0xffffffffu) {
				b = atomicAdd(&tcnt[part[k]], (unsigned int)__popc(m));
			}
			rank[k] = __shfl_sync(0xffffffffu, b, leader) + __popc(m & ((1u << lane) - 1));
		}
		__syncthreads();
		if (warp == 0) {
			uint32_t c = lane < nparts ? tcnt[lane] : 0, incl = c;
#pragma unroll
			for (int d = 1; d < PF_MAXP; d <<= 1) {
				uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
				if (lane >= d) {
					incl += t;
				}
			}
			if (lane < nparts) {
				pstart[lane] = incl - c;
				base[lane] = c ? atomicAdd(&cursors[lane], (unsigned long long)c) : 0ULL;
			}
			if (lane == nparts - 1) {
				pstart[nparts] = incl;
			}
			if (BULK) {
				// re-lay the runs so that run p starts at a position with the parity of its global start
				__syncwarp();
				if (lane == 0) {
					uint32_t off = 0;
					for (int p = 0; p < nparts; p++) {
						off += (off ^ (uint32_t)base[p]) & 1u;
						pstart[p] = off;
						off += tcnt[p];
					}
					pstart[nparts] = off;
				}
			}
		}
		__syncthreads();
#pragma unroll
		for (int k = 0; k < PF_ROWS; k++) {
			if (part[k] != 0xffffffffu) {
				const uint32_t lp = pstart[part[k]] + rank[k];
				if (!BULK) {
					ppart[lp] = (uint8_t)part[k];
				}
#pragma unroll
				for (int c = 0; c < NC; c++) {
					stage[(size_t)c * CS + lp] = v[k][c];
				}
			}
		}
		if (BULK) {
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // generic-proxy writes -> visible to the bulk copies
		}
		__syncthreads();
		if (BULK) {
			if ((int)threadIdx.x < nparts * NC) {
				const int p = (int)threadIdx.x / NC, c = (int)threadIdx.x % NC;
				uint32_t len = tcnt[p];
				const uint64_t b = base[p];
				if (PEER && len && b + len > capacity) {
					// a receive buffer too small for this exchange: never write past it; the host reads the count and raises
					const uint32_t fit = b < capacity ? (uint32_t)(capacity - b) : 0u;
					if (c == 0) {
						atomicAdd(dropped, (unsigned long long)(len - fit));
					}
					len = fit;
				}
				if (len) {
					uint64_t *gd = (uint64_t *)(PEER ? dst.out[p][c] : pc.out[c]) + b;
					const uint64_t *ss = stage + (size_t)c * CS + pstart[p];
					const uint32_t head = (uint32_t)(b & 1ULL);
					if (head) {
						gd[0] = ss[0];
					}
					const uint32_t mid = (len - head) & ~1u;
					if (mid) {
						pf_bulk_store(gd + head, ss + head, mid * 8u);
					}
					if ((len - head) & 1u) {
						gd[len - 1] = ss[len - 1];
					}
				}
				asm volatile("cp.async.bulk.commit_group;" ::: "memory");
				asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); // the staged tile may be overwritten
			}
		} else {
#pragma unroll
			for (int k = 0; k < PF_ROWS; k++) {
				const uint32_t i = k * PF_THREADS + threadIdx.x;
				if (i >= rows_in_tile) {
					continue;
				}
				const uint32_t p = ppart[i];
				const uint64_t pos = base[p] + (i - pstart[p]);
				if (PEER && pos >= capacity) {
					atomicAdd(dropped, 1ULL); // a receive buffer too small for this exchange: never write past it
					continue;
				}
#pragma unroll
				for (int c = 0; c < NC; c++) {
					uint64_t *out = (uint64_t *)(PEER ? dst.out[p][c] : pc.out[c]);
					out[pos] = stage[(size_t)c * CS + i];
				}
			}
		}
		__syncthreads();
	}
	if (BULK) {
		asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); // all bulk writes of this thread have completed
	}
}

// columns permuted so that the key column comes first; false when the shape is not the register kernel's
static bool part_reg_shape(const KeyCols &keys, const PartCols &pc, const PartDst &dst, bool peer, int nparts, PartCols *rpc,
                           PartDst *rdst) {
	if (getenv("B200_PART_NO_REG") || !keys_fast64(keys) || pc.n < 1 || pc.n > 4) {
		return false;
	}
	int kc = -1;
	for (int c = 0; c < pc.n; c++) {
		if (pc.width[c] != 8) {
			return false;
		}
		if (pc.in[c] == keys.c[0].data) {
			kc = c;
		}
	}
	if (kc < 0) {
		return false;
	}
	*rpc = pc;
	*rdst = dst;
	std::swap(rpc->in[0], rpc->in[kc]);
	std::swap(rpc->out[0], rpc->out[kc]);
	if (peer) {
		for (int p = 0; p < nparts; p++) {
			std::swap(rdst->out[p][0], rdst->out[p][kc]);
		}
	}
	return true;
}

template <bool PEER, int NC, bool BULK>
static int launch_part_reg_v(b200_ctx *ctx, const PartCols &pc, const PartDst &dst, uint64_t n, int bits,
                             unsigned long long *cursors, uint64_t capacity, unsigned long long *dropped) {
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(part_move_reg_kernel<PEER, NC, BULK>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
		attr_set = true;
	}
	const size_t tile = (size_t)PF_THREADS * PF_ROWS;
	size_t smem = BULK ? (size_t)NC * (tile + PF_PAD) * 8 : (size_t)NC * tile * 8 + tile;
	uint64_t tiles = (n + tile - 1) / tile;
	uint64_t mg = (uint64_t)ctx->sm_count * 2;
	part_move_reg_kernel<PEER, NC, BULK><<<(unsigned)(tiles < mg ? tiles : mg), PF_THREADS, smem, ctx->stream>>>(
	    pc, dst, n, bits, cursors, capacity, dropped);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// B200_PART_BULK=1: runs leave shared memory by bulk-async copies (experimental until measured on NVLink)
template <bool PEER, int NC>
static int launch_part_reg(b200_ctx *ctx, const PartCols &pc, const PartDst &dst, uint64_t n, int bits,
                           unsigned long long *cursors, uint64_t capacity, unsigned long long *dropped) {
	const char *env = getenv("B200_PART_BULK"); // read per call: the tests flip it inside one process
	const bool bulk = env && atoi(env) != 0;
	if (bulk) {
		return launch_part_reg_v<PEER, NC, true>(ctx, pc, dst, n, bits, cursors, capacity, dropped);
	}
	return launch_part_reg_v<PEER, NC, false>(ctx, pc, dst, n, bits, cursors, capacity, dropped);
}

template <bool PEER>
static int launch_part_move(b200_ctx *ctx, const KeyCols &keys, const PartCols &pc, const PartDst &dst, uint64_t n, int bits,
                            unsigned long long *cursors, size_t stage_bytes, uint64_t capacity = ~0ULL,
                            unsigned long long *dropped = nullptr) {
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(part_move_staged_kernel<PEER, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(part_move_staged_kernel<PEER, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
		attr_set = true;
	}
	{
		PartCols rpc;
		PartDst rdst;
		if (part_reg_shape(keys, pc, dst, PEER, 1 << bits, &rpc, &rdst)) {
			switch (rpc.n) {
			case 1:
				return launch_part_reg<PEER, 1>(ctx, rpc, rdst, n, bits, cursors, capacity, dropped);
			case 2:
				return launch_part_reg<PEER, 2>(ctx, rpc, rdst, n, bits, cursors, capacity, dropped);
			case 3:
				return launch_part_reg<PEER, 3>(ctx, rpc, rdst, n, bits, cursors, capacity, dropped);
			default:
				return launch_part_reg<PEER, 4>(ctx, rpc, rdst, n, bits, cursors, capacity, dropped);
			}
		}
	}
	int mgrid = grid_for(n, PF_THREADS, PF_ROWS, ctx->sm_count * 8);
	size_t smem = stage_bytes + (size_t)PF_THREADS * PF_ROWS; // + the partition byte of every staged position
	if (keys_fast64(keys)) {
		part_move_staged_kernel<PEER, true><<<mgrid, PF_THREADS, smem, ctx->stream>>>(keys, pc, dst, n, bits, cursors, capacity, dropped);
	} else {
		part_move_staged_kernel<PEER, false><<<mgrid, PF_THREADS, smem, ctx->stream>>>(keys, pc, dst, n, bits, cursors, capacity, dropped);
	}
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

static void launch_part_count(b200_ctx *ctx, const KeyCols &keys, uint64_t n, int bits, unsigned long long *counts) {
	int fgrid = grid_for(n, PF_THREADS, 16, ctx->sm_count * 8);
	if (keys_fast64(keys)) {
		part_count_kernel<true><<<fgrid, PF_THREADS, 0, ctx->stream>>>(keys, n, bits, counts);
	} else {
		part_count_kernel<false><<<fgrid, PF_THREADS, 0, ctx->stream>>>(keys, n, bits, counts);
	}
	ctx->launches++;
}

extern "C" {

int b200_hash(b200_ctx *ctx, const b200_batch *b, const int *key_cols, int nkeys, uint64_t *out_hashes) {
	if (!ctx || !b || !key_cols || !out_hashes) {
		b200_set_error("b200_hash: bad arguments");
		return B200_ERR_INVALID;
	}
	KeyCols keys;
	B200_TRY(b200_fill_keycols(b, key_cols, nkeys, &keys, "b200_hash"));
	if (b->nrows == 0) {
		return B200_OK;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	int grid = grid_for(b->nrows, 256, 4, ctx->sm_count * 8);
	hash_kernel<<<grid, 256, 0, ctx->stream>>>(keys, b->nrows, out_hashes);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

int b200_radix_partition(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                         b200_batch **out, uint64_t *counts_host) {
	if (!ctx || !in || !key_cols || !out || !counts_host) {
		b200_set_error("b200_radix_partition: bad arguments");
		return B200_ERR_INVALID;
	}
	if (bits < 0 || bits > 12) {
		b200_set_error("b200_radix_partition: bits must be in [0,12] (radix_partitioning.hpp MAX_RADIX_BITS)");
		return B200_ERR_INVALID;
	}
	if (in->nrows > 0xffffffffULL) {
		b200_set_error("b200_radix_partition: at most 2^32-1 rows per batch");
		return B200_ERR_INVALID;
	}
	// both paths move values as at most 8 bytes (the fast path's width switch, store_raw / col_load_raw)
	for (size_t ci = 0; ci < in->cols.size(); ci++) {
		if (in->cols[ci].type == B200_INT128) {
			b200_set_error("b200_radix_partition: INT128 columns are not supported (column %d)", (int)ci);
			return B200_ERR_INVALID;
		}
	}
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, nkeys, &keys, "b200_radix_partition"));
	CUDA_TRY(cudaSetDevice(ctx->device));
	int nparts = 1 << bits;
	uint64_t n = in->nrows;
	b200_batch *ob = b200_batch_new(ctx, n);
	// fast path: few partitions (the GPU-level shuffle: bits = log2(#GPUs)), flat columns without NULLs
	bool fast = bits <= 4 && (int)in->cols.size() <= TP_MAX_PART_COLS && n > 0 && !getenv("B200_PART_GENERIC");
	size_t fast_row_bytes = 0;
	for (size_t ci = 0; ci < in->cols.size() && fast; ci++) {
		fast = in->cols[ci].vtype == B200_FLAT_VECTOR && !in->cols[ci].validity;
		fast_row_bytes += (size_t)b200_type_size(in->cols[ci].type);
	}
	fast = fast && fast_row_bytes * PF_THREADS * PF_ROWS <= 96 * 1024;
	if (fast) {
		unsigned long long *cc = nullptr;
		int r0 = b200_dev_alloc(ctx, 2 * PF_MAXP * 8, (void **)&cc);
		if (r0 != B200_OK) {
			b200_batch_free(ob);
			return r0;
		}
		unsigned long long *fcounts = cc, *fcursors = cc + PF_MAXP;
		cudaMemsetAsync(cc, 0, 2 * PF_MAXP * 8, ctx->stream);
		PartCols pc;
		pc.n = (int)in->cols.size();
		for (int ci = 0; ci < pc.n; ci++) {
			void *data = nullptr;
			r0 = b200_batch_add_flat(ob, in->cols[ci].type, n, false, &data, nullptr);
			if (r0 != B200_OK) {
				b200_dev_free(ctx, cc);
				b200_batch_free(ob);
				return r0;
			}
			pc.in[ci] = in->cols[ci].data;
			pc.out[ci] = data;
			pc.width[ci] = b200_type_size(in->cols[ci].type);
		}
		launch_part_count(ctx, keys, n, bits, fcounts);
		exclusive_scan_small_kernel<<<1, 32, 0, ctx->stream>>>(fcounts, fcursors, nparts);
		ctx->launches++;
		PartDst no_dst;
		memset(&no_dst, 0, sizeof(no_dst));
		int mr = launch_part_move<false>(ctx, keys, pc, no_dst, n, bits, fcursors, fast_row_bytes * PF_THREADS * PF_ROWS);
		if (mr != B200_OK) {
			b200_dev_free(ctx, cc);
			b200_batch_free(ob);
			return mr;
		}
		cudaError_t fe = cudaMemcpyAsync(counts_host, fcounts, nparts * 8, cudaMemcpyDeviceToHost, ctx->stream);
		ctx->d2h_bytes += nparts * 8;
		b200_dev_free(ctx, cc);
		fe = fe ? fe : cudaStreamSynchronize(ctx->stream);
		fe = fe ? fe : cudaGetLastError();
		if (fe != cudaSuccess) {
			b200_batch_free(ob);
			return b200_cuda_fail(fe, "radix_partition(fast)", __FILE__, __LINE__);
		}
		*out = ob;
		return B200_OK;
	}
	unsigned long long *counts = nullptr, *cursors = nullptr;
	uint32_t *part_of_row = nullptr, *dest = nullptr;
	int r = b200_dev_alloc(ctx, nparts * 8, (void **)&counts);
	r = r ? r : b200_dev_alloc(ctx, nparts * 8, (void **)&cursors);
	r = r ? r : b200_dev_alloc(ctx, (n + 1) * 4, (void **)&part_of_row);
	r = r ? r : b200_dev_alloc(ctx, (n + 1) * 4, (void **)&dest);
	auto free_scratch = [&]() {
		b200_dev_free(ctx, counts);
		b200_dev_free(ctx, cursors);
		b200_dev_free(ctx, part_of_row);
		b200_dev_free(ctx, dest);
	};
	if (r != B200_OK) {
		free_scratch();
		b200_batch_free(ob);
		return r;
	}
	cudaMemsetAsync(counts, 0, nparts * 8, ctx->stream);
	int grid = grid_for(n ? n : 1, 256, 8, ctx->sm_count * 4);
	if (n) {
		part_hist_kernel<<<grid, 256, nparts * 4, ctx->stream>>>(keys, n, bits, counts, part_of_row);
		ctx->launches++;
	}
	exclusive_scan_small_kernel<<<1, 32, 0, ctx->stream>>>(counts, cursors, nparts);
	ctx->launches++;
	if (n) {
		size_t sh = (size_t)(nparts + (nparts & 1)) * 4 + (size_t)nparts * 8;
		part_scatter_index_kernel<<<grid, 256, sh, ctx->stream>>>(part_of_row, n, bits, cursors, dest);
		ctx->launches++;
	}
	for (size_t ci = 0; ci < in->cols.size(); ci++) {
		const DCol &c = in->cols[ci];
		void *data = nullptr;
		uint64_t *val = nullptr;
		r = b200_batch_add_flat(ob, c.type, n, c.validity != nullptr, &data, &val);
		if (r != B200_OK) {
			free_scratch();
			b200_batch_free(ob);
			return r;
		}
		if (n) {
			if (val) {
				uint64_t words = (n + 63) / 64;
				fill_u64_kernel<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(val, words, ~0ULL);
				ctx->launches++;
			}
			part_scatter_col_kernel<<<grid, 256, 0, ctx->stream>>>(c, n, dest, data, val);
			ctx->launches++;
		}
	}
	// counts can exceed the 64-word scratch: copy directly (pageable destination is fine, we sync)
	cudaError_t e = cudaMemcpyAsync(counts_host, counts, nparts * 8, cudaMemcpyDeviceToHost, ctx->stream);
	ctx->d2h_bytes += nparts * 8;
	b200_dev_free(ctx, counts);
	b200_dev_free(ctx, cursors);
	b200_dev_free(ctx, part_of_row);
	b200_dev_free(ctx, dest);
	if (e != cudaSuccess) {
		b200_batch_free(ob);
		return b200_cuda_fail(e, "cudaMemcpyAsync(counts)", __FILE__, __LINE__);
	}
	e = cudaStreamSynchronize(ctx->stream);
	if (e == cudaSuccess) {
		e = cudaGetLastError();
	}
	if (e != cudaSuccess) {
		b200_batch_free(ob);
		return b200_cuda_fail(e, "radix_partition", __FILE__, __LINE__);
	}
	*out = ob;
	return B200_OK;
}

// ---------------------------------------------------------------- shuffle without an intermediate copy (experimental)
static int part_fast_eligible(const b200_batch *in, int bits, PartCols *pc, size_t *stage_bytes, const char *who) {
	if (bits < 0 || bits > 4 || (int)in->cols.size() > TP_MAX_PART_COLS || in->cols.empty()) {
		b200_set_error("%s: needs 0..4 radix bits and 1..%d columns", who, TP_MAX_PART_COLS);
		return B200_ERR_INVALID;
	}
	size_t row_bytes = 0;
	pc->n = (int)in->cols.size();
	for (int ci = 0; ci < pc->n; ci++) {
		const DCol &c = in->cols[ci];
		if (c.vtype != B200_FLAT_VECTOR || c.validity) {
			b200_set_error("%s: column %d must be a flat vector without NULLs", who, ci);
			return B200_ERR_INVALID;
		}
		if (c.type == B200_INT128) {
			// the move kernels copy values of 1, 2, 4 or 8 bytes
			b200_set_error("%s: INT128 columns are not supported (column %d)", who, ci);
			return B200_ERR_INVALID;
		}
		pc->in[ci] = c.data;
		pc->out[ci] = nullptr;
		pc->width[ci] = b200_type_size(c.type);
		row_bytes += (size_t)pc->width[ci];
	}
	*stage_bytes = row_bytes * PF_THREADS * PF_ROWS;
	if (*stage_bytes > 96 * 1024) {
		b200_set_error("%s: rows of %zu bytes do not fit the staging tile", who, row_bytes);
		return B200_ERR_INVALID;
	}
	return B200_OK;
}

int b200_partition_count(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                         uint64_t *counts_host) {
	if (!ctx || !in || !key_cols || !counts_host) {
		b200_set_error("b200_partition_count: bad arguments");
		return B200_ERR_INVALID;
	}
	PartCols pc;
	size_t stage_bytes = 0;
	B200_TRY(part_fast_eligible(in, bits, &pc, &stage_bytes, "b200_partition_count"));
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, nkeys, &keys, "b200_partition_count"));
	CUDA_TRY(cudaSetDevice(ctx->device));
	int nparts = 1 << bits;
	for (int p = 0; p < nparts; p++) {
		counts_host[p] = 0;
	}
	uint64_t n = in->nrows;
	if (n == 0) {
		return B200_OK;
	}
	unsigned long long *counts = nullptr;
	B200_TRY(b200_dev_alloc(ctx, PF_MAXP * 8, (void **)&counts));
	cudaMemsetAsync(counts, 0, PF_MAXP * 8, ctx->stream);
	launch_part_count(ctx, keys, n, bits, counts);
	cudaError_t e = cudaMemcpyAsync(counts_host, counts, nparts * 8, cudaMemcpyDeviceToHost, ctx->stream);
	ctx->d2h_bytes += nparts * 8;
	b200_dev_free(ctx, counts);
	e = e ? e : cudaStreamSynchronize(ctx->stream);
	e = e ? e : cudaGetLastError();
	if (e != cudaSuccess) {
		return b200_cuda_fail(e, "partition_count", __FILE__, __LINE__);
	}
	return B200_OK;
}

int b200_partition_scatter(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                           void *const *dst_cols, const uint64_t *dst_row_offsets) {
	if (!ctx || !in || !key_cols || !dst_cols || !dst_row_offsets) {
		b200_set_error("b200_partition_scatter: bad arguments");
		return B200_ERR_INVALID;
	}
	PartCols pc;
	size_t stage_bytes = 0;
	B200_TRY(part_fast_eligible(in, bits, &pc, &stage_bytes, "b200_partition_scatter"));
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, nkeys, &keys, "b200_partition_scatter"));
	CUDA_TRY(cudaSetDevice(ctx->device));
	int nparts = 1 << bits;
	uint64_t n = in->nrows;
	if (n == 0) {
		return B200_OK;
	}
	PartDst dst;
	memset(&dst, 0, sizeof(dst));
	for (int p = 0; p < nparts; p++) {
		for (int c = 0; c < pc.n; c++) {
			dst.out[p][c] = dst_cols[p * pc.n + c];
			if (!dst.out[p][c]) {
				b200_set_error("b200_partition_scatter: destination of partition %d, column %d is NULL", p, c);
				return B200_ERR_INVALID;
			}
		}
	}
	unsigned long long *cursors = nullptr;
	B200_TRY(b200_dev_alloc(ctx, PF_MAXP * 8, (void **)&cursors));
	// the per-partition cursors start at the caller's row offsets (where this source's rows go in each destination)
	for (int p = 0; p < PF_MAXP; p++) {
		ctx->pinned_scratch[44 + p] = p < nparts ? dst_row_offsets[p] : 0;
	}
	cudaError_t e = cudaMemcpyAsync(cursors, ctx->pinned_scratch + 44, PF_MAXP * 8, cudaMemcpyHostToDevice, ctx->stream);
	int mr = B200_OK;
	if (e == cudaSuccess) {
		mr = launch_part_move<true>(ctx, keys, pc, dst, n, bits, cursors, stage_bytes);
	}
	b200_dev_free(ctx, cursors);
	// the pinned scratch words are re-used by the next call: wait for the copy (and the kernel) before returning
	e = e ? e : cudaStreamSynchronize(ctx->stream);
	if (e != cudaSuccess) {
		return b200_cuda_fail(e, "partition_scatter", __FILE__, __LINE__);
	}
	return mr;
}

// Stream-asynchronous variants for a shuffle without host round trips (duckdb_b200/distributed.py PeerShuffle):
// counts and write offsets stay in device memory, nothing synchronises.
int b200_partition_count_dev(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                             uint64_t *counts_dev) {
	if (!ctx || !in || !key_cols || !counts_dev) {
		b200_set_error("b200_partition_count_dev: bad arguments");
		return B200_ERR_INVALID;
	}
	PartCols pc;
	size_t stage_bytes = 0;
	B200_TRY(part_fast_eligible(in, bits, &pc, &stage_bytes, "b200_partition_count_dev"));
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, nkeys, &keys, "b200_partition_count_dev"));
	CUDA_TRY(cudaSetDevice(ctx->device));
	CUDA_TRY(cudaMemsetAsync(counts_dev, 0, (size_t)(1 << bits) * 8, ctx->stream));
	if (in->nrows) {
		launch_part_count(ctx, keys, in->nrows, bits, (unsigned long long *)counts_dev);
	}
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

int b200_partition_scatter_dev(b200_ctx *ctx, const b200_batch *in, const int *key_cols, int nkeys, int bits,
                               void *const *dst_cols, const uint64_t *dst_row_offsets_dev, uint64_t capacity_rows,
                               uint64_t *dropped_dev) {
	if (!ctx || !in || !key_cols || !dst_cols || !dst_row_offsets_dev || !dropped_dev) {
		b200_set_error("b200_partition_scatter_dev: bad arguments");
		return B200_ERR_INVALID;
	}
	PartCols pc;
	size_t stage_bytes = 0;
	B200_TRY(part_fast_eligible(in, bits, &pc, &stage_bytes, "b200_partition_scatter_dev"));
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, nkeys, &keys, "b200_partition_scatter_dev"));
	CUDA_TRY(cudaSetDevice(ctx->device));
	int nparts = 1 << bits;
	uint64_t n = in->nrows;
	if (n == 0) {
		return B200_OK;
	}
	PartDst dst;
	memset(&dst, 0, sizeof(dst));
	for (int p = 0; p < nparts; p++) {
		for (int c = 0; c < pc.n; c++) {
			dst.out[p][c] = dst_cols[p * pc.n + c];
			if (!dst.out[p][c]) {
				b200_set_error("b200_partition_scatter_dev: destination of partition %d, column %d is NULL", p, c);
				return B200_ERR_INVALID;
			}
		}
	}
	// the kernel advances the cursors: work on a copy of the caller's offsets
	unsigned long long *cursors = nullptr;
	B200_TRY(b200_dev_alloc(ctx, PF_MAXP * 8, (void **)&cursors));
	cudaError_t e = cudaMemcpyAsync(cursors, dst_row_offsets_dev, (size_t)nparts * 8, cudaMemcpyDeviceToDevice, ctx->stream);
	int mr = B200_OK;
	if (e == cudaSuccess) {
		mr = launch_part_move<true>(ctx, keys, pc, dst, n, bits, cursors, stage_bytes, capacity_rows,
		                            (unsigned long long *)dropped_dev);
	}
	b200_dev_free(ctx, cursors); // stream-ordered: released after the kernel
	if (e != cudaSuccess) {
		return b200_cuda_fail(e, "partition_scatter_dev", __FILE__, __LINE__);
	}
	return mr;
}

} // extern "C"
