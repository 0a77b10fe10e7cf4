// RIGHT / FULL OUTER joins: the build-side half.  The probe kernels (join.cu, join_tile.cu) flag every build row they
// emit; b200_join_scan_unmatched (join.cu) compacts the unflagged rows of a range through b200_filter_project.  The
// compaction returns row ids relative to the range, and this kernel turns them into build row ids.
#include "join.cuh"

__global__ void __launch_bounds__(256) join_rows_offset_kernel(uint32_t *__restrict__ rows, uint64_t n, uint32_t base) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
		rows[i] += base;
	}
}

int b200_join_rows_offset_launch(b200_ctx *ctx, uint32_t *rows, uint64_t n, uint32_t base) {
	join_rows_offset_kernel<<<grid_for(n, 256, 4, ctx->sm_count * 8), 256, 0, ctx->stream>>>(rows, n, base);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}
