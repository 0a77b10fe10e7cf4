// Shared device/host definitions for the operator kernels (H100, sm_90a).
// Layout notes live in DESIGN.md ("Data layout in HBM").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/duckdb_b200.h"

#define B200_SM_COUNT 132 // H100 SXM; only a fallback, the context reads the device attribute

// ----------------------------------------------------------------- errors
void b200_set_error(const char *fmt, ...);
int b200_cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define CUDA_TRY(expr)                                                                                                 \
	do {                                                                                                               \
		cudaError_t _e = (expr);                                                                                       \
		if (_e != cudaSuccess) {                                                                                       \
			return b200_cuda_fail(_e, #expr, __FILE__, __LINE__);                                                      \
		}                                                                                                              \
	} while (0)

#define B200_TRY(expr)                                                                                                 \
	do {                                                                                                               \
		int _r = (expr);                                                                                               \
		if (_r != B200_OK) {                                                                                           \
			return _r;                                                                                                 \
		}                                                                                                              \
	} while (0)

// ----------------------------------------------------------------- device column view
// Device-side mirror of b200_vector (= UnifiedVectorFormat).  All pointers are device pointers.
struct DCol {
	const void *data;
	const uint32_t *sel;
	const uint64_t *validity;
	int32_t type;
	int32_t vtype;
};

struct b200_ctx {
	int device;
	cudaStream_t stream;
	bool own_stream;
	int sm_count;
	uint64_t launches;
	uint64_t h2d_bytes;
	uint64_t d2h_bytes;
	// small pinned scratch for counters read back by the host
	uint64_t *pinned_scratch; // 64 words
	// device scratch for counters
	uint64_t *dev_scratch; // 64 words
	size_t l2_persist_max;  // bytes of L2 that may be set aside for persisting accesses (0 = unsupported)
	size_t l2_window_max;   // largest access-policy window
	size_t l2_size;         // bytes of L2 (cudaDevAttrL2CacheSize; 50 MB on an H100 SXM)
};

// Pin [ptr, ptr+bytes) in L2 for the kernels launched next on the context's stream (hash tables that are re-used
// by every probe / sink row); b200_l2_unpin resets the stream's window.
void b200_l2_pin(b200_ctx *ctx, const void *ptr, size_t bytes);
void b200_l2_unpin(b200_ctx *ctx);

struct b200_batch {
	b200_ctx *ctx;
	uint64_t nrows;
	std::vector<DCol> cols;
	std::vector<uint64_t> dict_sizes;
	std::vector<void *> owned; // device allocations freed with the batch
};

int b200_dev_alloc(b200_ctx *ctx, size_t bytes, void **out);
void b200_dev_free(b200_ctx *ctx, void *p);
b200_batch *b200_batch_new(b200_ctx *ctx, uint64_t nrows);
// allocate a flat output column (data + optional validity) owned by `b`
int b200_batch_add_flat(b200_batch *b, int type, uint64_t capacity_rows, bool with_validity, void **data,
                        uint64_t **validity);

static inline __host__ __device__ int b200_type_size(int t) {
	switch (t) {
	case B200_BOOL:
	case B200_UINT8:
	case B200_INT8:
		return 1;
	case B200_UINT16:
	case B200_INT16:
		return 2;
	case B200_UINT32:
	case B200_INT32:
	case B200_FLOAT:
		return 4;
	case B200_UINT64:
	case B200_INT64:
	case B200_DOUBLE:
		return 8;
	case B200_INT128:
		return 16;
	default:
		return 0;
	}
}

static inline __host__ __device__ bool b200_type_is_signed_int(int t) {
	return t == B200_INT8 || t == B200_INT16 || t == B200_INT32 || t == B200_INT64;
}
static inline __host__ __device__ bool b200_type_is_unsigned_int(int t) {
	return t == B200_BOOL || t == B200_UINT8 || t == B200_UINT16 || t == B200_UINT32 || t == B200_UINT64;
}
static inline __host__ __device__ bool b200_type_is_integer(int t) {
	return b200_type_is_signed_int(t) || b200_type_is_unsigned_int(t);
}
static inline __host__ __device__ bool b200_type_is_float(int t) {
	return t == B200_FLOAT || t == B200_DOUBLE;
}

#ifdef __CUDACC__
// ----------------------------------------------------------------- device helpers

// streaming (read-once) loads: keep them out of L1 (guide: Guideline 13/14)
template <class T>
__device__ __forceinline__ T ld_stream(const T *p) {
	return __ldcs(p);
}

__device__ __forceinline__ uint64_t col_index(const DCol &c, uint64_t row) {
	if (c.vtype == B200_FLAT_VECTOR) {
		return row;
	}
	if (c.vtype == B200_CONSTANT_VECTOR) {
		return 0;
	}
	return c.sel[row];
}

__device__ __forceinline__ bool col_valid_at(const DCol &c, uint64_t idx) {
	if (!c.validity) {
		return true;
	}
	return (c.validity[idx >> 6] >> (idx & 63)) & 1;
}

// Load value `idx` widened to 64 bits: signed types sign-extended, unsigned zero-extended,
// float -> its 32 bits (zero-extended), double -> its 64 bits.
__device__ __forceinline__ uint64_t col_load_raw(const DCol &c, uint64_t idx) {
	switch (c.type) {
	case B200_BOOL:
	case B200_UINT8:
		return ((const uint8_t *)c.data)[idx];
	case B200_INT8:
		return (uint64_t)(int64_t)((const int8_t *)c.data)[idx];
	case B200_UINT16:
		return ((const uint16_t *)c.data)[idx];
	case B200_INT16:
		return (uint64_t)(int64_t)((const int16_t *)c.data)[idx];
	case B200_UINT32:
	case B200_FLOAT:
		return ((const uint32_t *)c.data)[idx];
	case B200_INT32:
		return (uint64_t)(int64_t)((const int32_t *)c.data)[idx];
	default:
		return ((const uint64_t *)c.data)[idx];
	}
}

__device__ __forceinline__ void store_raw(void *dst, int type, uint64_t i, uint64_t v) {
	switch (b200_type_size(type)) {
	case 1:
		((uint8_t *)dst)[i] = (uint8_t)v;
		break;
	case 2:
		((uint16_t *)dst)[i] = (uint16_t)v;
		break;
	case 4:
		((uint32_t *)dst)[i] = (uint32_t)v;
		break;
	default:
		((uint64_t *)dst)[i] = v;
		break;
	}
}

// duckdb::MurmurHash64 (src/include/duckdb/common/types/hash.hpp:38-45)
__host__ __device__ __forceinline__ uint64_t murmur64(uint64_t x) {
	x ^= x >> 32;
	x *= 0xd6e8feb86659fd93ULL;
	x ^= x >> 32;
	x *= 0xd6e8feb86659fd93ULL;
	x ^= x >> 32;
	return x;
}

#define B200_NULL_HASH 0xbf58476d1ce4e5b9ULL

// duckdb::Hash<T>(value) on a raw widened value (hash.hpp:47-54; hash.cpp:33-57):
// integers narrower than 64 bits hash their uint32 cast; -0.0 -> +0.0, NaN -> canonical quiet NaN.
__host__ __device__ __forceinline__ uint64_t hash_raw(int type, uint64_t raw) {
	switch (type) {
	case B200_UINT64:
	case B200_INT64:
		return murmur64(raw);
	case B200_DOUBLE: {
		uint64_t bits = raw;
		if ((bits << 1) == 0) {
			bits = 0; // +-0.0
		} else if ((bits & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL) {
			bits = 0x7ff8000000000000ULL; // NaN
		}
		return murmur64(bits);
	}
	case B200_FLOAT: {
		uint32_t bits = (uint32_t)raw;
		if ((bits << 1) == 0) {
			bits = 0;
		} else if ((bits & 0x7fffffffu) > 0x7f800000u) {
			bits = 0x7fc00000u;
		}
		return murmur64((uint64_t)bits);
	}
	default:
		return murmur64((uint64_t)(uint32_t)raw);
	}
}

// CombineHashScalar (vector_hash.cpp:44-48)
__host__ __device__ __forceinline__ uint64_t combine_hash(uint64_t a, uint64_t b) {
	a ^= a >> 32;
	a *= 0xd6e8feb86659fd93ULL;
	return a ^ b;
}

// Canonical key bits for equality: two values are "the same group / join key" iff these are equal.
// Floats: -0.0 == +0.0, all NaNs equal (comparison_operators.cpp:24-40).
__device__ __forceinline__ uint64_t canonical_key_bits(int type, uint64_t raw) {
	if (type == B200_DOUBLE) {
		if ((raw << 1) == 0) {
			return 0;
		}
		if ((raw & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL) {
			return 0x7ff8000000000000ULL;
		}
		return raw;
	}
	if (type == B200_FLOAT) {
		uint32_t bits = (uint32_t)raw;
		if ((bits << 1) == 0) {
			return 0;
		}
		if ((bits & 0x7fffffffu) > 0x7f800000u) {
			return 0x7fc00000u;
		}
		return bits;
	}
	return raw;
}

#define MAX_KEYS 8
struct KeyCols {
	DCol c[MAX_KEYS];
	int n;
};

// hash of the key columns of one row; *any_null set if a key is NULL
__device__ __forceinline__ uint64_t hash_row(const KeyCols &k, uint64_t row, bool *any_null) {
	uint64_t h = 0;
	bool nul = false;
#pragma unroll 1
	for (int j = 0; j < k.n; j++) {
		uint64_t idx = col_index(k.c[j], row);
		bool valid = col_valid_at(k.c[j], idx);
		uint64_t hv = valid ? hash_raw(k.c[j].type, col_load_raw(k.c[j], idx)) : B200_NULL_HASH;
		nul |= !valid;
		h = (j == 0) ? hv : combine_hash(h, hv);
	}
	*any_null = nul;
	return h;
}

static inline int grid_for(uint64_t n, int threads, int rows_per_thread, int max_blocks) {
	uint64_t per_block = (uint64_t)threads * rows_per_thread;
	uint64_t blocks = (n + per_block - 1) / per_block;
	if (blocks < 1) {
		blocks = 1;
	}
	if (blocks > (uint64_t)max_blocks) {
		blocks = max_blocks;
	}
	return (int)blocks;
}
#endif // __CUDACC__
