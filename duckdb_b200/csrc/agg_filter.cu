// Filtered aggregates (FILTER (WHERE ...), and the filtered aggregates DuckDB binds a small PIVOT to): the validity fold.
//
// DuckDB extracts an aggregate's filter into the projection below the aggregate as a BOOLEAN column of the child
// chunk (plan_aggregate.cpp:342-348).  The hash aggregate still creates the group of every row, but updates a
// filtered aggregate only with the rows where that column is TRUE; NULL and FALSE skip it
// (physical_hash_aggregate.cpp:361-404,442-466).  For every function the sink supports that is exactly "the input is
// NULL where the filter is not TRUE": SUM / MIN / MAX / AVG over no rows are NULL, COUNT over no rows is 0.  So the
// fold turns each (input, filter) pair into an input with a validity mask, and the sink paths, which already take
// nullable inputs, run unchanged:
//
//   bit i of pair j's validity = input valid at row i AND filter valid at row i AND filter byte != 0
//
// One launch covers every filtered pair of a b200_agg_sink call (blockIdx.y = pair).  Input and filter are read
// through their selection, so FLAT, CONSTANT and DICTIONARY vectors all work.  A dictionary's (or a constant's)
// validity is indexed by its own positions, so a per-row mask cannot be attached to it: such an input is also gathered
// into a flat scratch column in the same pass.  A FLAT input keeps its data pointer and only gets the new validity,
// so the tile paths stage its data once however many filters read it.  A warp handles 32 consecutive rows at a time
// and stores their validity bits with one ballot (half of a 64-bit validity_t word), like join_mark.cu.
#include "agg.cuh"
#include <cstring>

#define AF_THREADS 256
#define AF_UNROLL 4 // 32-row slices per warp and step: their loads are issued back to back

struct FoldPair {
	DCol in;
	DCol filt;
	uint32_t *valid32; // the output validity words as 32-bit halves
	void *gather;      // flat copy of a non-FLAT input (nullptr: the input is FLAT and keeps its data)
	int width;         // bytes per input value
};

struct FoldArgs {
	FoldPair p[MAX_INPUTS];
	uint64_t n;
};

__device__ __forceinline__ void af_copy(void *dst, const void *src, uint64_t row, uint64_t idx, int width) {
	switch (width) {
	case 1:
		((uint8_t *)dst)[row] = ((const uint8_t *)src)[idx];
		break;
	case 2:
		((uint16_t *)dst)[row] = ((const uint16_t *)src)[idx];
		break;
	case 4:
		((uint32_t *)dst)[row] = ((const uint32_t *)src)[idx];
		break;
	default:
		((uint64_t *)dst)[row] = ((const uint64_t *)src)[idx];
		break;
	}
}

__global__ void __launch_bounds__(AF_THREADS) agg_filter_fold_kernel(const __grid_constant__ FoldArgs A) {
	const FoldPair &P = A.p[blockIdx.y];
	const uint64_t n = A.n;
	const int lane = threadIdx.x & 31;
	const uint64_t warps = (uint64_t)gridDim.x * (AF_THREADS / 32);
	const uint64_t step = warps * 32 * AF_UNROLL;
	for (uint64_t base = ((uint64_t)blockIdx.x * AF_THREADS + threadIdx.x) / 32 * (32 * AF_UNROLL); base < n;
	     base += step) {
		bool pass[AF_UNROLL];
#pragma unroll
		for (int k = 0; k < AF_UNROLL; k++) {
			uint64_t row = base + k * 32 + lane;
			pass[k] = false;
			if (row < n) {
				uint64_t fi = col_index(P.filt, row), ii = col_index(P.in, row);
				pass[k] = col_valid_at(P.filt, fi) && ((const uint8_t *)P.filt.data)[fi] != 0 && col_valid_at(P.in, ii);
				if (P.gather) {
					af_copy(P.gather, P.in.data, row, ii, P.width);
				}
			}
		}
#pragma unroll
		for (int k = 0; k < AF_UNROLL; k++) {
			uint32_t bits = __ballot_sync(0xffffffffu, pass[k]);
			uint64_t row0 = base + k * 32;
			if (lane == 0 && row0 < n) {
				P.valid32[row0 >> 5] = bits;
			}
		}
	}
}

// bytes of one scratch region: 256-byte aligned, so the tile paths can bulk-copy it
static size_t fold_span(size_t bytes) {
	return (bytes + 255) & ~(size_t)255;
}

// Enqueue the fold of npairs (input, filter) pairs over n >= 1 rows (filters already checked to be B200_BOOL).  out[j]
// is pair j's input as a FLAT column with the folded validity.  *scratch receives the one device block the outputs
// live in: the caller frees it (stream-ordered) after the kernels that read them.
int b200_agg_filter_fold(b200_ctx *ctx, const DCol *in, const DCol *filt, int npairs, uint64_t n, DCol *out,
                         void **scratch) {
	*scratch = nullptr;
	if (npairs <= 0) {
		return B200_OK;
	}
	const size_t vbytes = fold_span(((n + 63) / 64) * 8);
	size_t total = 0;
	for (int j = 0; j < npairs; j++) {
		total += vbytes;
		if (in[j].vtype != B200_FLAT_VECTOR) {
			total += fold_span((size_t)n * b200_type_size(in[j].type));
		}
	}
	void *block = nullptr;
	B200_TRY(b200_dev_alloc(ctx, total, &block));
	FoldArgs A;
	memset(&A, 0, sizeof(A));
	A.n = n;
	unsigned char *p = (unsigned char *)block;
	for (int j = 0; j < npairs; j++) {
		FoldPair &P = A.p[j];
		P.in = in[j];
		P.filt = filt[j];
		P.width = b200_type_size(in[j].type);
		P.valid32 = (uint32_t *)p;
		p += vbytes;
		out[j] = in[j];
		out[j].validity = (const uint64_t *)P.valid32;
		if (in[j].vtype != B200_FLAT_VECTOR) {
			P.gather = p;
			p += fold_span((size_t)n * P.width);
			out[j].data = P.gather;
			out[j].sel = nullptr;
			out[j].vtype = B200_FLAT_VECTOR;
		}
	}
	const uint64_t rows_per_block = (uint64_t)AF_THREADS * AF_UNROLL;
	uint64_t blocks = (n + rows_per_block - 1) / rows_per_block;
	uint64_t max_blocks = (uint64_t)ctx->sm_count * 8;
	dim3 grid((unsigned)(blocks < max_blocks ? blocks : max_blocks), (unsigned)npairs);
	agg_filter_fold_kernel<<<grid, AF_THREADS, 0, ctx->stream>>>(A);
	ctx->launches++;
	*scratch = block;
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) {
		b200_dev_free(ctx, block);
		*scratch = nullptr;
		return b200_cuda_fail(e, "agg_filter_fold_kernel", __FILE__, __LINE__);
	}
	return B200_OK;
}
