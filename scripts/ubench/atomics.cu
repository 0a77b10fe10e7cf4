// Micro-benchmark: random-access primitives the aggregate / join tables are built from, as a function of the table
// size (L2-resident vs HBM).  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench/_build/atomics
// scripts/ubench/atomics.cu ; run on an H100: scripts/ubench/_build/atomics [ops_millions]
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

__device__ __forceinline__ uint64_t mix(uint64_t x) {
	x ^= x >> 32;
	x *= 0xd6e8feb86659fd93ULL;
	x ^= x >> 32;
	x *= 0xd6e8feb86659fd93ULL;
	x ^= x >> 32;
	return x;
}

__device__ __forceinline__ void red64(uint64_t *p, uint64_t v) {
	asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// MODE 0: red, 1: ld16 + red same sector, 2: ld16 + 2 red same sector, 3: ld16 (sector 0) + red (sector 1, needs stride>=8),
// 4: returning atomicAdd, 5: ld16 only, 6: st8 only, 7: ld16 + returning atomic + red, 8: 4 x red same 32B sector... etc.
template <int MODE, int ROWS>
__global__ void __launch_bounds__(256) k(uint64_t *tab, uint64_t mask, int stride_words, uint64_t n, uint64_t *sink) {
	uint64_t acc = 0;
	uint64_t i0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * ROWS;
	uint64_t step = (uint64_t)gridDim.x * blockDim.x * ROWS;
	for (uint64_t i = i0; i < n; i += step) {
		uint64_t *row[ROWS];
#pragma unroll
		for (int r = 0; r < ROWS; r++) {
			row[r] = tab + (mix(i + r) & mask) * (uint64_t)stride_words;
		}
		if (MODE == 1 || MODE == 2 || MODE == 3 || MODE == 5 || MODE == 7) {
			ulonglong2 v[ROWS];
#pragma unroll
			for (int r = 0; r < ROWS; r++) {
				asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(v[r].x), "=l"(v[r].y) : "l"(row[r]) : "memory");
			}
#pragma unroll
			for (int r = 0; r < ROWS; r++) {
				acc += v[r].x ^ v[r].y;
			}
		}
#pragma unroll
		for (int r = 0; r < ROWS; r++) {
			if (MODE == 0 || MODE == 1 || MODE == 2 || MODE == 8) {
				red64(row[r] + 2, i);
			}
			if (MODE == 2 || MODE == 8) {
				red64(row[r] + 3, 1);
			}
			if (MODE == 8) {
				red64(row[r] + 0, 1);
				red64(row[r] + 1, 1);
			}
			if (MODE == 3) {
				red64(row[r] + 4, i);
			}
			if (MODE == 4 || MODE == 7) {
				acc += atomicAdd((unsigned long long *)(row[r] + 2), (unsigned long long)i);
			}
			if (MODE == 7) {
				red64(row[r] + 3, 1);
			}
			if (MODE == 6) {
				row[r][2] = i;
			}
		}
	}
	if (acc == 0x1234567) {
		*sink = acc;
	}
}

template <int MODE>
static void run(const char *name, uint64_t *tab, size_t bytes, int stride_words, uint64_t n, uint64_t *sink) {
	uint64_t slots = bytes / (stride_words * 8);
	uint64_t mask = slots - 1;
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0);
	cudaEventCreate(&e1);
	int grid = 132 * 8; // 8 CTAs per SM of an H100 SXM
	k<MODE, 4><<<grid, 256>>>(tab, mask, stride_words, n / 4, sink);
	cudaEventRecord(e0);
	k<MODE, 4><<<grid, 256>>>(tab, mask, stride_words, n, sink);
	cudaEventRecord(e1);
	cudaEventSynchronize(e1);
	float ms = 0;
	cudaEventElapsedTime(&ms, e0, e1);
	cudaError_t e = cudaGetLastError();
	printf("%-34s table %6zu MB stride %3d B : %8.3f ms  %7.2f G rows/s %s\n", name, bytes >> 20, stride_words * 8, ms,
	       n / ms / 1e6, e == cudaSuccess ? "" : cudaGetErrorString(e));
	fflush(stdout);
}

int main(int argc, char **argv) {
	uint64_t n = (argc > 1 ? atoll(argv[1]) : 256) * 1000000ULL;
	size_t maxb = 4ULL << 30;
	uint64_t *tab, *sink;
	cudaMalloc(&tab, maxb);
	cudaMalloc(&sink, 8);
	cudaMemset(tab, 0, maxb);
	size_t sizes[] = {16ULL << 20, 64ULL << 20, 128ULL << 20, 256ULL << 20, 1ULL << 30, 4ULL << 30};
	for (size_t b : sizes) {
		run<5>("ld16", tab, b, 4, n, sink);
		run<6>("st8", tab, b, 4, n, sink);
		run<0>("red64", tab, b, 4, n, sink);
		run<1>("ld16+red64 (same sector)", tab, b, 4, n, sink);
		run<2>("ld16+2xred64 (same sector)", tab, b, 4, n, sink);
		run<8>("4xred64 (same sector)", tab, b, 4, n, sink);
		run<3>("ld16+red64 (next sector)", tab, b, 8, n, sink);
		run<4>("atom64 returning", tab, b, 4, n, sink);
		run<7>("ld16+atom64+red64", tab, b, 4, n, sink);
		run<2>("ld16+2xred64 stride 128", tab, b, 16, n, sink);
	}
	return 0;
}
