// K3 join_build + K4 join_probe.
// Reference semantics: JoinHashTable::Build / Finalize / InsertHashesLoop / Probe / ScanStructure::Next* /
// GatherRHS (src/execution/join_hashtable.cpp:617-712,1113-1139,858-984,1178-1209,1476-2300,1690-1730),
// PhysicalHashJoin::{Sink,Finalize,ExecuteInternal} (src/execution/operator/join/physical_hash_join.cpp:764,1893,2140).
// NULL keys never match (join_hashtable.cpp:714-742); float keys: -0.0 == +0.0, NaN == NaN.
//
// Design (GPU-first, not the reference's salted pointer table over a row store):
//   * build rows live in a COLUMNAR device store (payload columns, flat);
//   * the hash table is open addressing with 16-byte slots {key64, head_row32, inline32}:
//       - one key column of <= 8 bytes: key64 is the canonical key itself -> a probe is ONE 32-byte sector,
//         no second dependent access to compare keys;
//       - composite keys: key64 is the 64-bit DuckDB hash; candidates are verified against the key store;
//   * duplicate build keys are chained through next[row] (the reference chains through an in-row pointer);
//   * when all build keys are unique and the payload fits 4 bytes it is ALSO kept inline in the slot, so the
//     probe of a PK-FK join (TPC-H Q14) never touches the payload store.
#include "join.cuh"
#include <cstring>
#include <cstdlib>

int b200_fill_keycols(const b200_batch *b, const int *cols, int n, KeyCols *out, const char *who);
int b200_join_probe_tile(b200_ctx *ctx, const JoinView &J, const KeyCols &keys, const ProbeOut &po, int join_type,
                         uint64_t n, uint64_t out_capacity, unsigned long long *counters);

// ------------------------------------------------------------------ build
__global__ void __launch_bounds__(256)
    join_append_kernel(KeyCols keys, bool exact, uint64_t n, uint64_t base, uint64_t *__restrict__ hashes,
                       uint8_t *__restrict__ row_skip, KeyStore ks, unsigned long long *__restrict__ counters) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		bool nul = false;
		uint64_t key64;
		if (exact) {
			const DCol &c = keys.c[0];
			uint64_t idx = col_index(c, row);
			nul = !col_valid_at(c, idx);
			key64 = canonical_key_bits(c.type, col_load_raw(c, idx));
		} else {
			key64 = hash_row(keys, row, &nul);
			for (int j = 0; j < keys.n; j++) {
				const DCol &c = keys.c[j];
				uint64_t idx = col_index(c, row);
				ks.data[j][base + row] = canonical_key_bits(c.type, col_load_raw(c, idx));
			}
		}
		hashes[base + row] = key64;
		row_skip[base + row] = nul ? 1 : 0;
		if (nul) {
			atomicAdd(&counters[2], 1ULL);
		}
	}
}

__global__ void __launch_bounds__(256)
    join_append_col_kernel(DCol c, uint64_t n, uint64_t base, void *__restrict__ out, uint64_t *__restrict__ out_valid) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		uint64_t idx = col_index(c, row);
		store_raw(out, c.type, base + row, col_load_raw(c, idx));
		if (out_valid && !col_valid_at(c, idx)) {
			uint64_t d = base + row;
			atomicAnd((unsigned long long *)&out_valid[d >> 6], ~(1ULL << (d & 63)));
		}
	}
}

__global__ void join_init_slots_kernel(JoinSlot *slots, uint64_t n) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
		slots[i].key = EMPTY_KEY;
		slots[i].head = ROW_NONE;
		slots[i].inl = 0;
	}
}

__global__ void __launch_bounds__(256)
    join_insert_kernel(JoinSlot *slots, uint64_t mask, bool exact, int key_type, const uint64_t *__restrict__ hashes,
                       const uint8_t *__restrict__ row_skip, uint64_t nrows, uint32_t *__restrict__ next,
                       unsigned long long *__restrict__ counters) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < nrows; row += stride) {
		if (row_skip[row]) {
			next[row] = ROW_NONE;
			continue;
		}
		uint64_t key = hashes[row];
		uint64_t slot;
		if (key == EMPTY_KEY) {
			slot = mask + 1; // side slot
		} else {
			slot = slot_hash(exact, key_type, key) & mask;
			while (true) {
				uint64_t k = *(volatile uint64_t *)&slots[slot].key;
				if (k == EMPTY_KEY) {
					unsigned long long old = atomicCAS((unsigned long long *)&slots[slot].key,
					                                   (unsigned long long)EMPTY_KEY, (unsigned long long)key);
					if (old == EMPTY_KEY || old == key) {
						break;
					}
				} else if (k == key) {
					break;
				}
				slot = (slot + 1) & mask;
			}
		}
		uint32_t old_head = atomicExch(&slots[slot].head, (uint32_t)row);
		next[row] = old_head;
		if (old_head != ROW_NONE) {
			atomicAdd(&counters[0], 1ULL);
		}
	}
}

// min / max of the build keys (canonical 64-bit values; signed or unsigned order)
__global__ void __launch_bounds__(256)
    join_minmax_kernel(const uint64_t *__restrict__ keys, const uint8_t *__restrict__ skip, uint64_t n, bool is_signed,
                       unsigned long long *__restrict__ out /* [0]=min, [1]=max, as ordered-uint64 */) {
	uint64_t lo = ~0ULL, hi = 0;
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	const uint64_t flip = is_signed ? (1ULL << 63) : 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
		if (skip[i]) {
			continue;
		}
		uint64_t v = keys[i] ^ flip;
		lo = v < lo ? v : lo;
		hi = v > hi ? v : hi;
	}
	for (int off = 16; off; off >>= 1) {
		uint64_t olo = __shfl_xor_sync(0xffffffffu, lo, off), ohi = __shfl_xor_sync(0xffffffffu, hi, off);
		lo = olo < lo ? olo : lo;
		hi = ohi > hi ? ohi : hi;
	}
	if ((threadIdx.x & 31) == 0) {
		atomicMin(&out[0], (unsigned long long)lo);
		atomicMax(&out[1], (unsigned long long)hi);
	}
}

// direct-addressed build: entry = row + 1, or (inline payload << 8) | 1; a second row for the same key sets dup
__global__ void __launch_bounds__(256)
    join_dense_build_kernel(uint32_t *__restrict__ dense, uint64_t dmin, const uint64_t *__restrict__ keys,
                            const uint8_t *__restrict__ skip, uint64_t n, bool inline_payload, PayloadStore ps,
                            unsigned long long *__restrict__ counters) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
		if (skip[row]) {
			continue;
		}
		uint32_t e = (uint32_t)row + 1;
		if (inline_payload) {
			uint32_t v = 0;
			int sh = 0;
			for (int p = 0; p < ps.n; p++) {
				int sz = b200_type_size(ps.type[p]);
				uint32_t raw = sz == 1 ? ((const uint8_t *)ps.data[p])[row] : ((const uint16_t *)ps.data[p])[row];
				v |= raw << sh;
				sh += sz * 8;
			}
			e = (v << 8) | 1u;
		}
		uint32_t old = atomicCAS(&dense[keys[row] - dmin], 0u, e);
		if (old != 0) {
			atomicAdd(&counters[0], 1ULL); // duplicate key: the dense table cannot be used
		}
	}
}

// unique build keys + payload <= 4 bytes: copy the payload bits of the head row into the slot
__global__ void __launch_bounds__(256) join_inline_kernel(JoinSlot *slots, uint64_t nslots, PayloadStore ps) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nslots; s += stride) {
		uint32_t r = slots[s].head;
		if (r == ROW_NONE) {
			continue;
		}
		uint32_t v = 0;
		int sh = 0;
		for (int p = 0; p < ps.n; p++) {
			int sz = b200_type_size(ps.type[p]);
			uint64_t raw = 0;
			switch (sz) {
			case 1:
				raw = ((const uint8_t *)ps.data[p])[r];
				break;
			case 2:
				raw = ((const uint16_t *)ps.data[p])[r];
				break;
			default:
				raw = ((const uint32_t *)ps.data[p])[r];
				break;
			}
			v |= (uint32_t)raw << sh;
			sh += sz * 8;
		}
		slots[s].inl = v;
	}
}

// MODE 0: count result rows only; MODE 1: write.  One warp-aggregated atomicAdd on the output cursor per
// warp iteration; a warp's results are written contiguously.
template <int MODE>
__global__ void __launch_bounds__(256)
    join_probe_kernel(JoinView J, KeyCols keys, ProbeOut po, int join_type, uint64_t n, uint64_t out_capacity,
                      unsigned long long *__restrict__ counters) {
	const int lane = threadIdx.x & 31;
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	uint64_t n_round = (n + 31) / 32 * 32;
	unsigned long long local_total = 0;
	for (uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_round; row += stride) {
		bool in_range = row < n;
		bool key_null = false;
		uint64_t ckeys[MAX_KEYS];
		uint32_t inl = 0;
		uint32_t first = ROW_NONE;
		if (in_range) {
			first = probe_first(J, keys, row, &key_null, ckeys, &inl);
		}
		uint32_t cnt = 0;
		if (in_range) {
			switch (join_type) {
			case B200_JOIN_INNER:
			case B200_JOIN_LEFT:
				if (first != ROW_NONE) {
					if (J.unique) {
						cnt = 1;
					} else {
						for (uint32_t r = first; r != ROW_NONE; r = chain_next(J, r, ckeys)) {
							cnt++;
						}
					}
				} else if (join_type == B200_JOIN_LEFT) {
					cnt = 1;
				}
				break;
			case B200_JOIN_SEMI:
				cnt = first != ROW_NONE;
				break;
			case B200_JOIN_ANTI:
				cnt = first == ROW_NONE;
				break;
			default: // MARK
				cnt = 1;
				break;
			}
		}
		if (MODE == 0) {
			local_total += cnt;
			continue;
		}
		// warp exclusive scan of cnt
		uint32_t incl = cnt;
#pragma unroll
		for (int off = 1; off < 32; off <<= 1) {
			uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
			if (lane >= off) {
				incl += t;
			}
		}
		uint32_t warp_total = __shfl_sync(0xffffffffu, incl, 31);
		unsigned long long base = 0;
		if (lane == 0 && warp_total) {
			base = atomicAdd(&counters[1], (unsigned long long)warp_total);
		}
		base = __shfl_sync(0xffffffffu, base, 0);
		if (!cnt) {
			continue;
		}
		uint64_t opos = base + incl - cnt;
		if (opos + cnt > out_capacity) {
			continue; // capacity exceeded: the host sees cursor > capacity and reports the error
		}
		switch (join_type) {
		case B200_JOIN_INNER:
		case B200_JOIN_LEFT:
			if (first == ROW_NONE) {
				emit_row(J, po, opos, row, ROW_NONE, 0, true);
			} else if (J.unique) {
				emit_row(J, po, opos, row, first, inl, true);
			} else {
				for (uint32_t r = first; r != ROW_NONE; r = chain_next(J, r, ckeys)) {
					emit_row(J, po, opos++, row, r, inl, true);
				}
			}
			break;
		case B200_JOIN_SEMI:
		case B200_JOIN_ANTI:
			emit_row(J, po, opos, row, ROW_NONE, 0, false);
			break;
		default: { // MARK: true if matched; NULL if the probe key is NULL or (no match and the build side has NULLs)
			emit_row(J, po, opos, row, ROW_NONE, 0, false);
			bool matched = first != ROW_NONE;
			po.mark[opos] = matched ? 1 : 0;
			if (!matched && (key_null || J.build_has_null) && !J.build_empty) {
				atomicAnd((unsigned long long *)&po.mark_valid[opos >> 6], ~(1ULL << (opos & 63)));
			}
			break;
		}
		}
	}
	if (MODE == 0) {
		for (int off = 16; off; off >>= 1) {
			local_total += __shfl_xor_sync(0xffffffffu, local_total, off);
		}
		if (lane == 0 && local_total) {
			atomicAdd(&counters[3], local_total);
		}
	}
}

__global__ void fill_u64_kernel4(uint64_t *p, uint64_t words, uint64_t v) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) {
		p[i] = v;
	}
}

// ------------------------------------------------------------------ host
static int join_reserve(b200_join *j, uint64_t need_rows) {
	if (need_rows <= j->capacity_rows) {
		return B200_OK;
	}
	b200_ctx *ctx = j->ctx;
	uint64_t cap = j->capacity_rows ? j->capacity_rows : 1024;
	while (cap < need_rows) {
		cap *= 2;
	}
	auto regrow = [&](void **p, size_t elem, bool fill_ones) -> int {
		void *np = nullptr;
		size_t old_bytes = (size_t)j->rows * elem;
		B200_TRY(b200_dev_alloc(ctx, (size_t)cap * elem + 16, &np));
		if (fill_ones) {
			cudaMemsetAsync(np, 0xff, (size_t)cap * elem + 16, ctx->stream);
		}
		if (*p && old_bytes) {
			CUDA_TRY(cudaMemcpyAsync(np, *p, old_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
		}
		b200_dev_free(ctx, *p);
		*p = np;
		return B200_OK;
	};
	B200_TRY(regrow((void **)&j->hashes, 8, false));
	B200_TRY(regrow((void **)&j->row_skip, 1, false));
	for (int k = 0; k < j->ks.n; k++) {
		B200_TRY(regrow((void **)&j->ks.data[k], 8, false));
	}
	for (int p = 0; p < j->ps.n; p++) {
		B200_TRY(regrow(&j->ps.data[p], b200_type_size(j->ps.type[p]), false));
		if (j->ps.validity[p]) {
			// validity bitmap: bytes = cap/8; copy old words
			void *np = nullptr;
			size_t nbytes = (cap + 63) / 64 * 8 + 16;
			B200_TRY(b200_dev_alloc(ctx, nbytes, &np));
			cudaMemsetAsync(np, 0xff, nbytes, ctx->stream);
			size_t old_bytes = (j->rows + 63) / 64 * 8;
			if (old_bytes) {
				CUDA_TRY(cudaMemcpyAsync(np, j->ps.validity[p], old_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
			}
			b200_dev_free(ctx, j->ps.validity[p]);
			j->ps.validity[p] = (uint64_t *)np;
		}
	}
	j->capacity_rows = cap;
	return B200_OK;
}

extern "C" {

int b200_join_create(b200_ctx *ctx, int join_type, const int32_t *key_types, int nkeys, const int32_t *payload_types,
                     int npayload, b200_join **out) {
	if (!ctx || !out || !key_types || nkeys < 1 || nkeys > MAX_KEYS || npayload < 0 || npayload > MAX_PAYLOAD ||
	    (npayload > 0 && !payload_types)) {
		b200_set_error("b200_join_create: bad arguments (1..%d keys, 0..%d payload columns)", MAX_KEYS, MAX_PAYLOAD);
		return B200_ERR_INVALID;
	}
	if (join_type != B200_JOIN_INNER && join_type != B200_JOIN_LEFT && join_type != B200_JOIN_SEMI &&
	    join_type != B200_JOIN_ANTI && join_type != B200_JOIN_MARK) {
		b200_set_error("b200_join_create: unsupported join type %d", join_type);
		return B200_ERR_INVALID;
	}
	b200_join *j = new b200_join();
	memset((void *)j, 0, sizeof(*j));
	j->ctx = ctx;
	j->join_type = join_type;
	j->nkeys = nkeys;
	for (int k = 0; k < nkeys; k++) {
		if (!b200_type_size(key_types[k]) || key_types[k] == B200_INT128) {
			b200_set_error("b200_join_create: unsupported key type %d", key_types[k]);
			delete j;
			return B200_ERR_INVALID;
		}
		j->key_type[k] = key_types[k];
	}
	j->exact = nkeys == 1;
	j->ks.n = j->exact ? 0 : nkeys;
	j->ps.n = npayload;
	for (int p = 0; p < npayload; p++) {
		if (!b200_type_size(payload_types[p]) || payload_types[p] == B200_INT128) {
			b200_set_error("b200_join_create: unsupported payload type %d", payload_types[p]);
			delete j;
			return B200_ERR_INVALID;
		}
		j->ps.type[p] = payload_types[p];
	}
	cudaSetDevice(ctx->device);
	void *p = nullptr;
	int rc = b200_dev_alloc(ctx, 64, &p);
	if (rc != B200_OK) {
		delete j;
		return rc;
	}
	j->counters = (unsigned long long *)p;
	cudaMemsetAsync(p, 0, 64, ctx->stream);
	*out = j;
	return B200_OK;
}

void b200_join_destroy(b200_join *j) {
	if (!j) {
		return;
	}
	b200_ctx *ctx = j->ctx;
	cudaSetDevice(ctx->device);
	b200_dev_free(ctx, j->hashes);
	b200_dev_free(ctx, j->row_skip);
	for (int k = 0; k < j->ks.n; k++) {
		b200_dev_free(ctx, j->ks.data[k]);
	}
	for (int p = 0; p < j->ps.n; p++) {
		b200_dev_free(ctx, j->ps.data[p]);
		b200_dev_free(ctx, j->ps.validity[p]);
	}
	b200_dev_free(ctx, j->slots);
	b200_dev_free(ctx, j->dense);
	b200_dev_free(ctx, j->next);
	b200_dev_free(ctx, j->counters);
	delete j;
}

int b200_join_build_sink(b200_join *j, const b200_batch *in, const int *key_cols, const int *payload_cols) {
	if (!j || !in || !key_cols || (j->ps.n > 0 && !payload_cols)) {
		b200_set_error("b200_join_build_sink: bad arguments");
		return B200_ERR_INVALID;
	}
	if (j->finalized) {
		b200_set_error("b200_join_build_sink: join is already finalized");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = j->ctx;
	KeyCols keys;
	B200_TRY(b200_fill_keycols(in, key_cols, j->nkeys, &keys, "b200_join_build_sink"));
	for (int k = 0; k < j->nkeys; k++) {
		if (keys.c[k].type != j->key_type[k]) {
			b200_set_error("b200_join_build_sink: key %d has type %d, join was created with %d", k, keys.c[k].type,
			               j->key_type[k]);
			return B200_ERR_INVALID;
		}
	}
	for (int p = 0; p < j->ps.n; p++) {
		if (payload_cols[p] < 0 || payload_cols[p] >= (int)in->cols.size() ||
		    in->cols[payload_cols[p]].type != j->ps.type[p]) {
			b200_set_error("b200_join_build_sink: payload column %d missing or of the wrong type", p);
			return B200_ERR_INVALID;
		}
	}
	uint64_t n = in->nrows;
	if (n == 0) {
		return B200_OK;
	}
	if (j->rows + n >= 0xffffffffULL) {
		b200_set_error("b200_join_build_sink: more than 2^32-2 build rows per GPU are not supported");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	// a payload column that gains a validity mask for the first time needs an all-valid bitmap for older rows
	for (int p = 0; p < j->ps.n; p++) {
		if (in->cols[payload_cols[p]].validity && !j->ps.validity[p]) {
			uint64_t cap = j->capacity_rows > j->rows + n ? j->capacity_rows : 0;
			(void)cap;
			size_t nbytes = ((j->capacity_rows ? j->capacity_rows : 1024) + 63) / 64 * 8 + 16;
			void *np = nullptr;
			B200_TRY(b200_dev_alloc(ctx, nbytes, &np));
			cudaMemsetAsync(np, 0xff, nbytes, ctx->stream);
			j->ps.validity[p] = (uint64_t *)np;
		}
	}
	if (j->capacity_rows == 0) {
		// first sink: the validity bitmaps above were sized for 1024 rows, which is what reserve starts with
	}
	B200_TRY(join_reserve(j, j->rows + n));
	int grid = grid_for(n, 256, 4, ctx->sm_count * 8);
	join_append_kernel<<<grid, 256, 0, ctx->stream>>>(keys, j->exact, n, j->rows, j->hashes, j->row_skip, j->ks,
	                                                  j->counters);
	ctx->launches++;
	for (int p = 0; p < j->ps.n; p++) {
		join_append_col_kernel<<<grid, 256, 0, ctx->stream>>>(in->cols[payload_cols[p]], n, j->rows, j->ps.data[p],
		                                                      j->ps.validity[p]);
		ctx->launches++;
	}
	CUDA_TRY(cudaGetLastError());
	j->rows += n;
	return B200_OK;
}

int b200_join_finalize(b200_join *j) {
	if (!j) {
		b200_set_error("b200_join_finalize: join is NULL");
		return B200_ERR_INVALID;
	}
	if (j->finalized) {
		return B200_OK;
	}
	b200_ctx *ctx = j->ctx;
	CUDA_TRY(cudaSetDevice(ctx->device));
	// Dense (direct-addressed) table: DuckDB's perfect hash join (perfect_hash_join_executor.cpp:70-133) for a
	// single integer key without duplicates whose range is small.  The reference caps the range at 1 M entries
	// (:121); here 4-byte entries live in HBM/L2, so the cap is the key density (range <= 8 x rows) and 1 GiB.
	if (j->exact && j->rows && b200_type_is_integer(j->key_type[0]) && !getenv("B200_JOIN_NO_DENSE")) {
		bool is_signed = b200_type_is_signed_int(j->key_type[0]);
		unsigned long long *mm = j->counters + 4;
		ctx->pinned_scratch[40] = ~0ULL;
		ctx->pinned_scratch[41] = 0;
		CUDA_TRY(cudaMemcpyAsync(mm, ctx->pinned_scratch + 40, 16, cudaMemcpyHostToDevice, ctx->stream));
		join_minmax_kernel<<<grid_for(j->rows, 256, 8, ctx->sm_count * 4), 256, 0, ctx->stream>>>(
		    j->hashes, j->row_skip, j->rows, is_signed, mm);
		ctx->launches++;
		CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 40, mm, 16, cudaMemcpyDeviceToHost, ctx->stream));
		CUDA_TRY(cudaStreamSynchronize(ctx->stream));
		uint64_t flip = is_signed ? (1ULL << 63) : 0;
		uint64_t omin = ctx->pinned_scratch[40], omax = ctx->pinned_scratch[41];
		if (omin <= omax) {
			uint64_t range = omax - omin + 1; // ordered-uint64 difference == key difference
			uint64_t limit = j->rows * 8 > (1ULL << 20) ? j->rows * 8 : (1ULL << 20);
			if (range != 0 && range <= limit && range <= (1ULL << 28)) {
				int pay_bytes = 0;
				bool pay_nullable = false;
				for (int p = 0; p < j->ps.n; p++) {
					pay_bytes += b200_type_size(j->ps.type[p]);
					pay_nullable = pay_nullable || j->ps.validity[p] != nullptr;
					if (b200_type_size(j->ps.type[p]) > 2) {
						pay_bytes = 99;
					}
				}
				bool inl = j->ps.n > 0 && pay_bytes <= 3 && !pay_nullable;
				uint32_t *dense = nullptr;
				B200_TRY(b200_dev_alloc(ctx, range * 4 + 16, (void **)&dense));
				CUDA_TRY(cudaMemsetAsync(dense, 0, range * 4, ctx->stream));
				CUDA_TRY(cudaMemsetAsync(j->counters, 0, 8, ctx->stream));
				uint64_t dmin = omin ^ flip; // back to the canonical key bits
				join_dense_build_kernel<<<grid_for(j->rows, 256, 4, ctx->sm_count * 8), 256, 0, ctx->stream>>>(
				    dense, dmin, j->hashes, j->row_skip, j->rows, inl, j->ps, j->counters);
				ctx->launches++;
				CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 24, j->counters, 4 * 8, cudaMemcpyDeviceToHost, ctx->stream));
				CUDA_TRY(cudaStreamSynchronize(ctx->stream));
				CUDA_TRY(cudaGetLastError());
				if (ctx->pinned_scratch[24] == 0) {
					j->dense = dense;
					j->dense_min = dmin;
					j->dense_range = range;
					j->unique = true;
					j->inline_payload = inl;
					j->has_null_key = ctx->pinned_scratch[26] != 0;
					b200_dev_free(ctx, j->hashes);
					j->hashes = nullptr;
					b200_dev_free(ctx, j->row_skip);
					j->row_skip = nullptr;
					j->finalized = true;
					return B200_OK;
				}
				b200_dev_free(ctx, dense); // duplicates: fall through to the hash table
				CUDA_TRY(cudaMemsetAsync(j->counters, 0, 8, ctx->stream));
			}
		}
	}
	// capacity: power of two >= 2 x rows (load factor <= 0.5), like JoinHashTable::PointerTableCapacity
	// (join_hashtable.hpp:565-577) but without its 16384 floor
	uint64_t cap = 1024;
	double max_load = 0.5;
	{
		const char *env = getenv("B200_JOIN_LOAD"); // experiment knob: maximum load factor of the table
		if (env && atof(env) > 0.05 && atof(env) < 0.95) {
			max_load = atof(env);
		}
	}
	while ((double)cap * max_load < (double)j->rows) {
		cap <<= 1;
	}
	j->table_cap = cap;
	B200_TRY(b200_dev_alloc(ctx, (cap + 1) * sizeof(JoinSlot), (void **)&j->slots));
	B200_TRY(b200_dev_alloc(ctx, (j->rows + 1) * 4, (void **)&j->next));
	join_init_slots_kernel<<<grid_for(cap + 1, 256, 4, ctx->sm_count * 8), 256, 0, ctx->stream>>>(j->slots, cap + 1);
	ctx->launches++;
	if (j->rows) {
		join_insert_kernel<<<grid_for(j->rows, 256, 2, ctx->sm_count * 8), 256, 0, ctx->stream>>>(
		    j->slots, cap - 1, j->exact, j->key_type[0], j->hashes, j->row_skip, j->rows, j->next, j->counters);
		ctx->launches++;
	}
	CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 24, j->counters, 4 * 8, cudaMemcpyDeviceToHost, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	CUDA_TRY(cudaGetLastError());
	ctx->d2h_bytes += 32;
	j->unique = ctx->pinned_scratch[24] == 0;
	j->has_null_key = ctx->pinned_scratch[26] != 0;
	int pay_bytes = 0;
	bool pay_nullable = false;
	for (int p = 0; p < j->ps.n; p++) {
		pay_bytes += b200_type_size(j->ps.type[p]);
		pay_nullable = pay_nullable || j->ps.validity[p] != nullptr;
	}
	// composite keys can collide on the 64-bit hash, so "no duplicates" is only exact for single keys
	j->inline_payload = j->unique && j->exact && j->ps.n > 0 && pay_bytes <= 4 && !pay_nullable;
	if (j->inline_payload && j->rows) {
		join_inline_kernel<<<grid_for(cap + 1, 256, 4, ctx->sm_count * 8), 256, 0, ctx->stream>>>(j->slots, cap + 1,
		                                                                                          j->ps);
		ctx->launches++;
	}
	if (!j->exact) {
		j->unique = false; // chains must be verified
	}
	// the per-row key64 array is only needed for insertion
	b200_dev_free(ctx, j->hashes);
	j->hashes = nullptr;
	b200_dev_free(ctx, j->row_skip);
	j->row_skip = nullptr;
	j->finalized = true;
	return B200_OK;
}

int b200_join_build_rows(b200_join *j, uint64_t *out_rows) {
	if (!j || !out_rows) {
		return B200_ERR_INVALID;
	}
	*out_rows = j->rows;
	return B200_OK;
}

int b200_join_probe(b200_join *j, const b200_batch *probe, const int *key_cols, const int *lhs_cols, int nlhs,
                    uint64_t out_capacity, b200_batch **out, uint32_t *out_lhs_sel, uint64_t *out_count) {
	if (!j || !probe || !key_cols || !out_count || nlhs < 0 || nlhs > MAX_LHS || (nlhs > 0 && !lhs_cols) || !out) {
		b200_set_error("b200_join_probe: bad arguments (at most %d lhs columns)", MAX_LHS);
		return B200_ERR_INVALID;
	}
	if (!j->finalized) {
		b200_set_error("b200_join_probe: call b200_join_finalize first");
		return B200_ERR_INVALID;
	}
	b200_ctx *ctx = j->ctx;
	KeyCols keys;
	B200_TRY(b200_fill_keycols(probe, key_cols, j->nkeys, &keys, "b200_join_probe"));
	for (int k = 0; k < j->nkeys; k++) {
		if (keys.c[k].type != j->key_type[k]) {
			b200_set_error("b200_join_probe: key %d has type %d, join was created with %d", k, keys.c[k].type,
			               j->key_type[k]);
			return B200_ERR_INVALID;
		}
	}
	for (int i = 0; i < nlhs; i++) {
		if (lhs_cols[i] < 0 || lhs_cols[i] >= (int)probe->cols.size()) {
			b200_set_error("b200_join_probe: lhs column index %d out of range", lhs_cols[i]);
			return B200_ERR_INVALID;
		}
	}
	uint64_t n = probe->nrows;
	if (n > 0xffffffffULL) {
		b200_set_error("b200_join_probe: at most 2^32-1 rows per batch");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	*out = nullptr;
	*out_count = 0;
	JoinView J;
	memset(&J, 0, sizeof(J));
	J.dense = j->dense;
	J.dense_min = j->dense_min;
	J.dense_range = j->dense_range;
	J.slots = j->slots;
	J.mask = j->table_cap - 1;
	J.next = j->next;
	J.exact = j->exact;
	J.unique = j->unique;
	J.inline_payload = j->inline_payload;
	J.nkeys = j->nkeys;
	for (int k = 0; k < j->nkeys; k++) {
		J.key_type[k] = j->key_type[k];
	}
	J.ks = j->ks;
	J.ps = j->ps;
	J.build_has_null = j->has_null_key;
	J.build_empty = j->rows == 0;
	int jt = j->join_type;
	bool with_payload = jt == B200_JOIN_INNER || jt == B200_JOIN_LEFT;
	ProbeOut po;
	memset(&po, 0, sizeof(po));
	po.nlhs = nlhs;
	po.lhs_sel = out_lhs_sel;
	int grid = grid_for(n ? n : 1, 256, 4, ctx->sm_count * 8);
	// result size: exact bound when every probe row yields at most one row, else a counting pass
	uint64_t cap = out_capacity;
	bool bounded = j->unique || jt == B200_JOIN_SEMI || jt == B200_JOIN_ANTI || jt == B200_JOIN_MARK;
	if (cap == 0) {
		if (bounded) {
			cap = n;
		} else if (n) {
			cudaMemsetAsync(j->counters + 3, 0, 8, ctx->stream);
			join_probe_kernel<0><<<grid, 256, 0, ctx->stream>>>(J, keys, po, jt, n, 0, j->counters);
			ctx->launches++;
			CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 32, j->counters + 3, 8, cudaMemcpyDeviceToHost, ctx->stream));
			CUDA_TRY(cudaStreamSynchronize(ctx->stream));
			CUDA_TRY(cudaGetLastError());
			ctx->d2h_bytes += 8;
			cap = ctx->pinned_scratch[32];
		}
	}
	b200_batch *ob = b200_batch_new(ctx, 0);
	int rc = B200_OK;
	uint64_t words = (cap + 63) / 64;
	auto fill_valid = [&](uint64_t *v) {
		if (v && words) {
			fill_u64_kernel4<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(v, words, ~0ULL);
			ctx->launches++;
		}
	};
	for (int i = 0; i < nlhs && rc == B200_OK; i++) {
		const DCol &c = probe->cols[lhs_cols[i]];
		po.lhs_src[i] = c;
		rc = b200_batch_add_flat(ob, c.type, cap, c.validity != nullptr, &po.lhs_data[i], &po.lhs_valid[i]);
		fill_valid(po.lhs_valid[i]);
	}
	if (with_payload) {
		for (int p = 0; p < j->ps.n && rc == B200_OK; p++) {
			bool nullable = j->ps.validity[p] != nullptr || jt == B200_JOIN_LEFT;
			rc = b200_batch_add_flat(ob, j->ps.type[p], cap, nullable, &po.pay_data[p], &po.pay_valid[p]);
			fill_valid(po.pay_valid[p]);
		}
	}
	if (jt == B200_JOIN_MARK && rc == B200_OK) {
		void *d;
		rc = b200_batch_add_flat(ob, B200_BOOL, cap, true, &d, &po.mark_valid);
		po.mark = (uint8_t *)d;
		fill_valid(po.mark_valid);
	}
	if (rc != B200_OK) {
		b200_batch_free(ob);
		return rc;
	}
	uint64_t count = 0;
	if (n) {
		cudaMemsetAsync(j->counters + 1, 0, 8, ctx->stream);
		// the table is re-used by every probe row: keep (as much as fits of) it in the persisting part of L2
		// (only when a good part of the table fits: pinning a small fraction of a large table slows the probe down)
		if (j->dense && j->dense_range * 4 <= 2 * ctx->l2_persist_max) {
			b200_l2_pin(ctx, j->dense, j->dense_range * 4);
		} else if (!j->dense && (j->table_cap + 1) * sizeof(JoinSlot) <= 2 * ctx->l2_persist_max) {
			b200_l2_pin(ctx, j->slots, (j->table_cap + 1) * sizeof(JoinSlot));
		}
		// TMA-staged probe when the batch is eligible (single key, flat aligned columns), else the generic kernel
		int trc = b200_join_probe_tile(ctx, J, keys, po, jt, n, cap, j->counters);
		if (trc == B200_ERR_INVALID) {
			join_probe_kernel<1><<<grid, 256, 0, ctx->stream>>>(J, keys, po, jt, n, cap, j->counters);
			ctx->launches++;
		} else if (trc != B200_OK) {
			b200_batch_free(ob);
			return trc;
		}
		cudaError_t e = cudaMemcpyAsync(ctx->pinned_scratch + 33, j->counters + 1, 8, cudaMemcpyDeviceToHost, ctx->stream);
		e = e ? e : cudaStreamSynchronize(ctx->stream);
		b200_l2_unpin(ctx); // after the kernel has finished: lines it would persist later are not covered by a reset
		e = e ? e : cudaGetLastError();
		if (e != cudaSuccess) {
			b200_batch_free(ob);
			return b200_cuda_fail(e, "join_probe", __FILE__, __LINE__);
		}
		ctx->d2h_bytes += 8;
		count = ctx->pinned_scratch[33];
	}
	if (count > cap) {
		b200_batch_free(ob);
		b200_set_error("b200_join_probe: %llu result rows exceed the output capacity %llu", (unsigned long long)count,
		               (unsigned long long)cap);
		return B200_ERR_CAPACITY;
	}
	ob->nrows = count;
	*out = ob;
	*out_count = count;
	return B200_OK;
}

} // extern "C"
