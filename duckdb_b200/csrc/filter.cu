// K5 filter_select + project.
// Reference semantics: PhysicalFilter::ExecuteInternal (src/execution/operator/filter/physical_filter.cpp:53-64),
// ExpressionExecutor::Select (src/execution/expression_executor.cpp:309-388), comparison selects
// (src/execution/expression_executor/execute_comparison.cpp:11-95), NULL/NaN comparison rules
// (src/include/duckdb/common/operator/comparison_operators.hpp:199-229,
//  src/common/vector_operations/comparison_operators.cpp:24-90), three-valued AND/OR
// (src/common/vector_operations/boolean_operators.cpp), DECIMAL arithmetic overflow
// (src/function/scalar/operator/arithmetic.cpp:975-1008, add.cpp:260, multiply.cpp:299).
//
// Three launches per batch (DESIGN.md "filter"):
//   A  filter_mask_kernel   evaluate predicate -> bitmask (DuckDB ValidityMask word layout) + per-tile popcounts
//   B  tile_scan_*_kernel   exclusive scan of the tile counts (three small coalesced launches)
//   C  compact_kernel       ordered compaction: evaluate projections for surviving rows, write them densely
#include "common.cuh"
#include <cstdlib>

#define MAX_NODES B200_MAX_EXPR_NODES
#define MAX_PCOLS 12
#define MAX_PROJ B200_MAX_PROJECTIONS
#define TILE_ROWS 2048 // rows per tile = 256 threads x 8

struct ExprProg {
	b200_expr_node nodes[MAX_NODES];
	DCol cols[MAX_PCOLS];
	int nnodes;
};

struct ProjOut {
	void *data[MAX_PROJ];
	uint64_t *validity[MAX_PROJ];
	int root[MAX_PROJ];
	int type[MAX_PROJ];
	int n;
};

__device__ __forceinline__ double raw_to_double(int type, uint64_t raw) {
	return type == B200_FLOAT ? (double)__uint_as_float((uint32_t)raw) : __longlong_as_double((long long)raw);
}

// three-way compare with DuckDB's total order on floats (NaN == NaN, NaN greater than everything)
__device__ __forceinline__ int compare_raw(int type, uint64_t a, uint64_t b) {
	if (b200_type_is_float(type)) {
		double x = raw_to_double(type, a), y = raw_to_double(type, b);
		bool xn = isnan(x), yn = isnan(y);
		if (xn || yn) {
			return xn && yn ? 0 : (xn ? 1 : -1);
		}
		return x < y ? -1 : (x > y ? 1 : 0);
	}
	if (b200_type_is_signed_int(type)) {
		int64_t x = (int64_t)a, y = (int64_t)b;
		return x < y ? -1 : (x > y ? 1 : 0);
	}
	return a < b ? -1 : (a > b ? 1 : 0);
}

__device__ __forceinline__ bool int_in_range(int type, int64_t v) {
	switch (type) {
	case B200_INT8:
		return v >= -128 && v <= 127;
	case B200_INT16:
		return v >= -32768 && v <= 32767;
	case B200_INT32:
		return v >= -2147483648LL && v <= 2147483647LL;
	case B200_UINT8:
		return v >= 0 && v <= 255;
	case B200_UINT16:
		return v >= 0 && v <= 65535;
	case B200_UINT32:
		return v >= 0 && v <= 4294967295LL;
	default:
		return true;
	}
}

// largest value of integer type t, as an unsigned 64-bit number
__device__ __forceinline__ uint64_t int_max(int t) {
	const int bits = b200_type_size(t) * 8;
	if (b200_type_is_signed_int(t)) {
		return (1ULL << (bits - 1)) - 1;
	}
	return bits == 64 ? ~0ULL : (1ULL << bits) - 1;
}

// Does the raw value s of an integer source (sign-extended when src_signed, zero-extended otherwise) lie in the range
// of integer type t?  TryCastWithOverflowCheck (numeric_cast.hpp) for every signedness pair and both 64-bit types.
__device__ __forceinline__ bool int_fits(int t, uint64_t s, bool src_signed) {
	if (src_signed && (int64_t)s < 0) {
		return b200_type_is_signed_int(t) && (int64_t)s >= -(int64_t)int_max(t) - 1;
	}
	return s <= int_max(t);
}

// the low bits of s that type t holds, sign- or zero-extended to 64 bits (the form eval_row keeps every raw value in)
__device__ __forceinline__ uint64_t extend_raw(int t, uint64_t s) {
	switch (t) {
	case B200_INT8:
		return (uint64_t)(int64_t)(int8_t)s;
	case B200_INT16:
		return (uint64_t)(int64_t)(int16_t)s;
	case B200_INT32:
		return (uint64_t)(int64_t)(int32_t)s;
	case B200_BOOL:
	case B200_UINT8:
		return (uint8_t)s;
	case B200_UINT16:
		return (uint16_t)s;
	case B200_UINT32:
		return (uint32_t)s;
	default:
		return s;
	}
}

__device__ __forceinline__ bool decimal_in_range(int type, int64_t v) {
	switch (type) {
	case B200_INT16:
		return v >= -9999 && v <= 9999;
	case B200_INT32:
		return v >= -999999999 && v <= 999999999;
	default:
		return v >= -999999999999999999LL && v <= 999999999999999999LL;
	}
}

// Evaluate the nodes whose bit is set in `need` (a dependency-closed set) for one row.  val/nul are per-thread arrays (local memory).
__device__ __forceinline__ void eval_row(const ExprProg &p, uint64_t row, uint32_t need, uint64_t *val, uint8_t *nul,
                                         int *overflow) {
#pragma unroll 1
	for (int i = 0; i < p.nnodes; i++) {
		if (!((need >> i) & 1u)) {
			continue;
		}
		const b200_expr_node &nd = p.nodes[i];
		uint64_t v = 0;
		bool isnull = false;
		switch (nd.op) {
		case B200_EXPR_COLREF: {
			const DCol &c = p.cols[nd.col];
			uint64_t idx = col_index(c, row);
			isnull = !col_valid_at(c, idx);
			v = col_load_raw(c, idx);
			break;
		}
		case B200_EXPR_CONST:
			v = nd.value.u;
			isnull = nd.is_null != 0;
			break;
		case B200_EXPR_NOT:
			isnull = nul[nd.left];
			v = !val[nd.left];
			break;
		case B200_EXPR_IS_NULL:
			v = nul[nd.left];
			break;
		case B200_EXPR_IS_NOT_NULL:
			v = !nul[nd.left];
			break;
		case B200_EXPR_EQ:
		case B200_EXPR_NE:
		case B200_EXPR_LT:
		case B200_EXPR_GT:
		case B200_EXPR_LE:
		case B200_EXPR_GE: {
			isnull = nul[nd.left] || nul[nd.right];
			int c = compare_raw(p.nodes[nd.left].type, val[nd.left], val[nd.right]);
			v = nd.op == B200_EXPR_EQ   ? c == 0
			    : nd.op == B200_EXPR_NE ? c != 0
			    : nd.op == B200_EXPR_LT ? c < 0
			    : nd.op == B200_EXPR_GT ? c > 0
			    : nd.op == B200_EXPR_LE ? c <= 0
			                            : c >= 0;
			break;
		}
		case B200_EXPR_DISTINCT:
		case B200_EXPR_NOT_DISTINCT: {
			bool ln = nul[nd.left], rn = nul[nd.right];
			bool distinct;
			if (ln || rn) {
				distinct = ln != rn;
			} else {
				distinct = compare_raw(p.nodes[nd.left].type, val[nd.left], val[nd.right]) != 0;
			}
			v = nd.op == B200_EXPR_DISTINCT ? distinct : !distinct;
			break;
		}
		case B200_EXPR_AND: {
			// FALSE dominates NULL
			bool ln = nul[nd.left], rn = nul[nd.right];
			bool lv = val[nd.left] != 0, rv = val[nd.right] != 0;
			if ((!ln && !lv) || (!rn && !rv)) {
				v = 0;
			} else if (ln || rn) {
				isnull = true;
			} else {
				v = 1;
			}
			break;
		}
		case B200_EXPR_OR: {
			// TRUE dominates NULL
			bool ln = nul[nd.left], rn = nul[nd.right];
			bool lv = val[nd.left] != 0, rv = val[nd.right] != 0;
			if ((!ln && lv) || (!rn && rv)) {
				v = 1;
			} else if (ln || rn) {
				isnull = true;
			} else {
				v = 0;
			}
			break;
		}
		case B200_EXPR_ADD:
		case B200_EXPR_SUB:
		case B200_EXPR_MUL: {
			isnull = nul[nd.left] || nul[nd.right];
			if (nd.type == B200_DOUBLE || nd.type == B200_FLOAT) {
				double x = raw_to_double(nd.type, val[nd.left]), y = raw_to_double(nd.type, val[nd.right]);
				double r = nd.op == B200_EXPR_ADD ? x + y : nd.op == B200_EXPR_SUB ? x - y : x * y;
				v = nd.type == B200_FLOAT ? (uint64_t)__float_as_uint((float)r)
				                          : (uint64_t)__double_as_longlong(r);
			} else {
				int64_t x = (int64_t)val[nd.left], y = (int64_t)val[nd.right];
				int64_t r;
				bool ovf = false;
				if (nd.op == B200_EXPR_ADD) {
					r = (int64_t)((uint64_t)x + (uint64_t)y);
					ovf = ((x ^ r) & (y ^ r)) < 0;
				} else if (nd.op == B200_EXPR_SUB) {
					r = (int64_t)((uint64_t)x - (uint64_t)y);
					ovf = ((x ^ y) & (x ^ r)) < 0;
				} else {
					r = (int64_t)((uint64_t)x * (uint64_t)y);
					int64_t hi = __mul64hi(x, y);
					ovf = hi != (r >> 63);
				}
				if (nd.type == B200_UINT64) {
					// unsigned 64-bit: recompute the overflow condition in unsigned arithmetic
					uint64_t ux = val[nd.left], uy = val[nd.right];
					if (nd.op == B200_EXPR_ADD) {
						ovf = ux + uy < ux;
					} else if (nd.op == B200_EXPR_SUB) {
						ovf = uy > ux;
					} else {
						ovf = __umul64hi(ux, uy) != 0;
					}
				}
				// nd.col: 0 = no check, 1 = range of the result type, 2 = DECIMAL bound of the result type
				if (nd.col == 1) {
					ovf = ovf || !int_in_range(nd.type, r);
				} else if (nd.col == 2) {
					ovf = ovf || !decimal_in_range(nd.type, r);
				} else {
					ovf = false;
				}
				if (ovf && !isnull) {
					*overflow = 1;
				}
				// unchecked results wrap to the width of their type (AddOperator etc.)
				v = extend_raw(nd.type, (uint64_t)r);
			}
			break;
		}
		case B200_EXPR_CAST: {
			// numeric cast with DuckDB's rules (TryCastWithOverflowCheck, numeric_cast.hpp): an integer must fit its
			// target, a 64-bit integer rounds once to FLOAT, a finite DOUBLE must stay finite as FLOAT, and any integer
			// becomes BOOL as `!= 0`.  FLOAT/DOUBLE -> integer is rejected by b200_filter_project.
			isnull = nul[nd.left];
			int st = p.nodes[nd.left].type;
			uint64_t s = val[nd.left];
			bool ovf = false;
			if (nd.type == B200_FLOAT) {
				float f;
				if (st == B200_DOUBLE) {
					double d = __longlong_as_double((long long)s);
					f = (float)d;
					ovf = isfinite(d) && isinf(f);
				} else if (st == B200_FLOAT) {
					f = __uint_as_float((uint32_t)s);
				} else if (b200_type_is_signed_int(st)) {
					f = __ll2float_rn((long long)s);
				} else {
					f = __ull2float_rn(s);
				}
				v = __float_as_uint(f);
			} else if (nd.type == B200_DOUBLE) {
				double d = b200_type_is_float(st)         ? raw_to_double(st, s)
				           : b200_type_is_signed_int(st) ? __ll2double_rn((long long)s)
				                                         : __ull2double_rn(s);
				v = (uint64_t)__double_as_longlong(d);
			} else if (nd.type == B200_BOOL) {
				v = s != 0;
			} else {
				ovf = !int_fits(nd.type, s, b200_type_is_signed_int(st));
				v = extend_raw(nd.type, s);
			}
			if (ovf && !isnull) {
				*overflow = 1;
			}
			break;
		}
		default:
			break;
		}
		val[i] = v;
		nul[i] = isnull;
	}
}

// A: predicate -> mask words (as uint32 halves) + per-tile counts.  One tile per block iteration.
__global__ void __launch_bounds__(256)
    filter_mask_kernel(ExprProg prog, int filter_root, uint32_t need, uint64_t n, uint32_t *__restrict__ mask32,
                       uint32_t *__restrict__ tile_counts, int *__restrict__ flags) {
	__shared__ uint32_t warp_cnt[8];
	uint64_t ntiles = (n + TILE_ROWS - 1) / TILE_ROWS;
	int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint64_t val[MAX_NODES];
	uint8_t nul[MAX_NODES];
	int overflow = 0;
	for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
		uint32_t cnt = 0;
#pragma unroll 2
		for (int k = 0; k < 8; k++) {
			// warp w handles groups w*8 .. w*8+7 of the tile (each group = 32 consecutive rows)
			uint64_t row = tile * TILE_ROWS + (uint64_t)(warp * 8 + k) * 32 + lane;
			bool keep = false;
			if (row < n) {
				eval_row(prog, row, need, val, nul, &overflow);
				keep = !nul[filter_root] && val[filter_root] != 0;
			}
			uint32_t m = __ballot_sync(0xffffffffu, keep);
			if (lane == 0 && tile * TILE_ROWS + (uint64_t)(warp * 8 + k) * 32 < n) {
				mask32[(tile * TILE_ROWS >> 5) + warp * 8 + k] = m;
			}
			cnt += __popc(m);
		}
		if (lane == 0) {
			warp_cnt[warp] = cnt;
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			uint32_t t = 0;
			for (int w = 0; w < 8; w++) {
				t += warp_cnt[w];
			}
			tile_counts[tile] = t;
		}
		__syncthreads();
	}
	if (overflow) {
		flags[0] = 1;
	}
}

// B: exclusive scan of the tile counts in three small coalesced launches:
//   B1 one CTA per chunk of 4096 tiles: local exclusive offsets + chunk total
//   B2 one CTA: exclusive scan of the chunk totals (-> chunk bases, grand total)
//   B3 add the chunk base to every local offset
#define SCAN_CHUNK 4096
__global__ void __launch_bounds__(1024)
    tile_scan_local_kernel(const uint32_t *__restrict__ counts, uint64_t *__restrict__ offsets, uint64_t ntiles,
                           uint64_t *__restrict__ chunk_totals) {
	__shared__ uint32_t warp_tot[32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	uint64_t base = (uint64_t)blockIdx.x * SCAN_CHUNK + (uint64_t)tid * 4;
	uint32_t c[4];
#pragma unroll
	for (int q = 0; q < 4; q++) {
		c[q] = base + q < ntiles ? counts[base + q] : 0;
	}
	uint32_t mine = c[0] + c[1] + c[2] + c[3];
	uint32_t incl = mine;
#pragma unroll
	for (int off = 1; off < 32; off <<= 1) {
		uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
		if (lane >= off) {
			incl += t;
		}
	}
	if (lane == 31) {
		warp_tot[warp] = incl;
	}
	__syncthreads();
	if (warp == 0) {
		uint32_t w = warp_tot[lane], wi = w;
#pragma unroll
		for (int off = 1; off < 32; off <<= 1) {
			uint32_t t = __shfl_up_sync(0xffffffffu, wi, off);
			if (lane >= off) {
				wi += t;
			}
		}
		warp_tot[lane] = wi - w; // exclusive prefix of the warp totals
		if (lane == 31) {
			chunk_totals[blockIdx.x] = wi;
		}
	}
	__syncthreads();
	uint64_t run = (uint64_t)warp_tot[warp] + incl - mine;
#pragma unroll
	for (int q = 0; q < 4; q++) {
		if (base + q < ntiles) {
			offsets[base + q] = run;
		}
		run += c[q];
	}
}

__global__ void __launch_bounds__(1024)
    tile_scan_chunks_kernel(uint64_t *__restrict__ chunk_totals, uint64_t nchunks, uint64_t *__restrict__ total_out) {
	// nchunks is small (n / 8 M rows): a serial scan by one thread is enough
	if (threadIdx.x == 0) {
		uint64_t run = 0;
		for (uint64_t i = 0; i < nchunks; i++) {
			uint64_t t = chunk_totals[i];
			chunk_totals[i] = run;
			run += t;
		}
		*total_out = run;
	}
}

__global__ void __launch_bounds__(1024)
    tile_scan_add_kernel(uint64_t *__restrict__ offsets, uint64_t ntiles, const uint64_t *__restrict__ chunk_bases) {
	uint64_t i = (uint64_t)blockIdx.x * SCAN_CHUNK + threadIdx.x;
	uint64_t b = chunk_bases[blockIdx.x];
#pragma unroll
	for (int q = 0; q < 4; q++, i += 1024) {
		if (i < ntiles) {
			offsets[i] += b;
		}
	}
}

// C: ordered compaction.  ALL = true: no filter, output position = row.
template <bool ALL>
__global__ void __launch_bounds__(256)
    compact_kernel(ExprProg prog, ProjOut po, uint32_t need, uint64_t n, const uint32_t *__restrict__ mask32,
                   const uint64_t *__restrict__ tile_offsets, uint32_t *__restrict__ out_sel,
                   int *__restrict__ flags) {
	__shared__ uint32_t group_base[64];
	uint64_t ntiles = (n + TILE_ROWS - 1) / TILE_ROWS;
	int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint64_t val[MAX_NODES];
	uint8_t nul[MAX_NODES];
	int overflow = 0;
	for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
		uint64_t tile_row0 = tile * TILE_ROWS;
		uint64_t out0 = ALL ? tile_row0 : tile_offsets[tile];
		if (!ALL) {
			// exclusive scan of the 64 group popcounts of this tile (two warps)
			if (threadIdx.x < 64) {
				uint64_t g_row = tile_row0 + (uint64_t)threadIdx.x * 32;
				uint32_t c = g_row < n ? __popc(mask32[(tile_row0 >> 5) + threadIdx.x]) : 0;
				uint32_t incl = c;
#pragma unroll
				for (int off = 1; off < 32; off <<= 1) {
					uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
					if (lane >= off) {
						incl += t;
					}
				}
				group_base[threadIdx.x] = incl - c;
			}
			__syncthreads();
			if (threadIdx.x >= 32 && threadIdx.x < 64) {
				// add the total of the first 32 groups to groups 32..63
				uint32_t last_base = group_base[31];
				uint64_t g_row = tile_row0 + 31ull * 32;
				uint32_t last_cnt = g_row < n ? __popc(mask32[(tile_row0 >> 5) + 31]) : 0;
				group_base[threadIdx.x] += last_base + last_cnt;
			}
			__syncthreads();
		}
#pragma unroll 1
		for (int k = 0; k < 8; k++) {
			int g = warp * 8 + k;
			uint64_t row = tile_row0 + (uint64_t)g * 32 + lane;
			bool keep;
			uint64_t opos;
			if (ALL) {
				keep = row < n;
				opos = row;
			} else {
				uint32_t m = (tile_row0 + (uint64_t)g * 32 < n) ? mask32[(tile_row0 >> 5) + g] : 0;
				keep = (m >> lane) & 1;
				opos = out0 + group_base[g] + __popc(m & ((1u << lane) - 1));
			}
			if (keep) {
				if (out_sel) {
					out_sel[opos] = (uint32_t)row;
				}
				if (po.n) {
					eval_row(prog, row, need, val, nul, &overflow);
					for (int j = 0; j < po.n; j++) {
						int r = po.root[j];
						store_raw(po.data[j], po.type[j], opos, val[r]);
						if (nul[r] && po.validity[j]) {
							atomicAnd((unsigned long long *)&po.validity[j][opos >> 6], ~(1ULL << (opos & 63)));
						}
					}
				}
			}
		}
		__syncthreads();
	}
	if (overflow) {
		flags[0] = 1;
	}
}

__global__ void fill_u64_kernel2(uint64_t *p, uint64_t words, uint64_t v) {
	uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) {
		p[i] = v;
	}
}

// filter_tile.cu: TMA-staged fast paths (return B200_ERR_INVALID when the expression shape is not eligible)
int b200_filter_mask_tile(b200_ctx *ctx, const b200_expr_node *nodes, int filter_root, const DCol *cols, int ncols,
                          uint64_t n, uint32_t *mask32, uint32_t *tile_counts);
int b200_filter_compact_tile(b200_ctx *ctx, const b200_expr_node *nodes, const int *proj_roots, int nproj,
                             void *const *out_data, const DCol *cols, int ncols, uint64_t n, const uint32_t *mask32,
                             const uint64_t *tile_offsets, uint32_t *out_sel);

static uint32_t closure_of(const ExprProg &p, uint32_t roots) {
	uint32_t need = roots;
	for (int i = p.nnodes - 1; i >= 0; i--) {
		if ((need >> i) & 1u) {
			if (p.nodes[i].left >= 0) {
				need |= 1u << p.nodes[i].left;
			}
			if (p.nodes[i].right >= 0) {
				need |= 1u << p.nodes[i].right;
			}
		}
	}
	return need;
}

static bool node_may_be_null(const ExprProg &p, int i, std::vector<int> &memo) {
	if (memo[i] >= 0) {
		return memo[i] != 0;
	}
	const b200_expr_node &nd = p.nodes[i];
	bool r;
	switch (nd.op) {
	case B200_EXPR_COLREF:
		r = p.cols[nd.col].validity != nullptr;
		break;
	case B200_EXPR_CONST:
		r = nd.is_null != 0;
		break;
	case B200_EXPR_IS_NULL:
	case B200_EXPR_IS_NOT_NULL:
	case B200_EXPR_DISTINCT:
	case B200_EXPR_NOT_DISTINCT:
		r = false;
		break;
	default:
		r = (nd.left >= 0 && node_may_be_null(p, nd.left, memo)) ||
		    (nd.right >= 0 && node_may_be_null(p, nd.right, memo));
		break;
	}
	memo[i] = r ? 1 : 0;
	return r;
}

int b200_filter_fused_tile(b200_ctx *ctx, const b200_expr_node *nodes, int filter_root, const int *proj_roots, int nproj,
                           void *const *out_data, const DCol *cols, int ncols, uint64_t n, uint32_t *mask32,
                           uint32_t *out_sel, uint32_t *status, unsigned long long *total_dev);

extern "C" int b200_filter_project(b200_ctx *ctx, const b200_batch *in, const b200_expr_node *nodes, int nnodes,
                                   int filter_root, const int *proj_roots, int nproj, b200_batch **out,
                                   uint32_t *out_sel, uint64_t *out_mask, uint64_t *out_count) {
	if (!ctx || !in || !out_count || (nnodes > 0 && !nodes) || (nproj > 0 && (!proj_roots || !out))) {
		b200_set_error("b200_filter_project: bad arguments");
		return B200_ERR_INVALID;
	}
	if (nnodes > MAX_NODES || nproj > MAX_PROJ || nnodes < 0 || nproj < 0) {
		b200_set_error("b200_filter_project: at most %d nodes and %d projections", MAX_NODES, MAX_PROJ);
		return B200_ERR_INVALID;
	}
	if (filter_root >= nnodes || filter_root < -1) {
		b200_set_error("b200_filter_project: filter_root out of range");
		return B200_ERR_INVALID;
	}
	ExprProg prog;
	prog.nnodes = nnodes;
	int col_map[256];
	int nmapped = 0;
	for (int i = 0; i < 256; i++) {
		col_map[i] = -1;
	}
	for (int i = 0; i < nnodes; i++) {
		prog.nodes[i] = nodes[i];
		const b200_expr_node &nd = nodes[i];
		if (nd.op == B200_EXPR_COLREF || nd.op == B200_EXPR_CONST) {
			prog.nodes[i].left = prog.nodes[i].right = -1;
		} else if (nd.op == B200_EXPR_NOT || nd.op == B200_EXPR_IS_NULL || nd.op == B200_EXPR_IS_NOT_NULL ||
		           nd.op == B200_EXPR_CAST) {
			prog.nodes[i].right = -1;
		}
		if ((nd.left >= i) || (nd.right >= i)) {
			b200_set_error("b200_filter_project: node %d references a later node (need topological order)", i);
			return B200_ERR_INVALID;
		}
		bool unary = nd.op == B200_EXPR_NOT || nd.op == B200_EXPR_IS_NULL || nd.op == B200_EXPR_IS_NOT_NULL ||
		             nd.op == B200_EXPR_CAST;
		bool leaf = nd.op == B200_EXPR_COLREF || nd.op == B200_EXPR_CONST;
		if (!leaf && (nd.left < 0 || (!unary && nd.right < 0))) {
			b200_set_error("b200_filter_project: node %d is missing an operand", i);
			return B200_ERR_INVALID;
		}
		if (!b200_type_size(nd.type) || nd.type == B200_INT128) {
			b200_set_error("b200_filter_project: node %d has unsupported type %d", i, nd.type);
			return B200_ERR_INVALID;
		}
		// Both operands of a comparison have one type (DuckDB binds them so) and an integer constant holds a value of
		// its type: the interpreter compares in the left operand's type, the tile path in the column's, and the two
		// only agree under these rules.
		if ((nd.op >= B200_EXPR_EQ && nd.op <= B200_EXPR_GE) || nd.op == B200_EXPR_DISTINCT ||
		    nd.op == B200_EXPR_NOT_DISTINCT) {
			if (nodes[nd.left].type != nodes[nd.right].type) {
				b200_set_error("b200_filter_project: node %d compares type %d with type %d", i, nodes[nd.left].type,
				               nodes[nd.right].type);
				return B200_ERR_INVALID;
			}
		}
		// DuckDB binds both operands of + - * to the result's type, and the interpreter reads them in that type.  The
		// check mode (`col`) is 0 (wrap), 1 (range of the type) or 2 (DECIMAL bound: INT16, INT32 and INT64 only).
		if (nd.op == B200_EXPR_ADD || nd.op == B200_EXPR_SUB || nd.op == B200_EXPR_MUL) {
			if (nd.type == B200_BOOL || nodes[nd.left].type != nd.type || nodes[nd.right].type != nd.type) {
				b200_set_error("b200_filter_project: node %d of type %d has operands of type %d and %d", i, nd.type,
				               nodes[nd.left].type, nodes[nd.right].type);
				return B200_ERR_INVALID;
			}
			bool decimal = nd.type == B200_INT16 || nd.type == B200_INT32 || nd.type == B200_INT64;
			if (!b200_type_is_float(nd.type) && (nd.col < 0 || nd.col > 2 || (nd.col == 2 && !decimal))) {
				b200_set_error("b200_filter_project: node %d has check mode %d for type %d", i, nd.col, nd.type);
				return B200_ERR_INVALID;
			}
		}
		// FLOAT/DOUBLE -> integer casts (rounding, range of the rounded value) are not implemented
		if (nd.op == B200_EXPR_CAST && b200_type_is_float(nodes[nd.left].type) && !b200_type_is_float(nd.type)) {
			b200_set_error("b200_filter_project: node %d casts type %d to type %d", i, nodes[nd.left].type, nd.type);
			return B200_ERR_INVALID;
		}
		if (nd.op == B200_EXPR_CONST && !nd.is_null && b200_type_is_integer(nd.type) && b200_type_size(nd.type) < 8) {
			const int bits = b200_type_size(nd.type) * 8;
			const int64_t v = nd.value.i;
			bool ok = b200_type_is_signed_int(nd.type) ? (v >= -(1LL << (bits - 1)) && v < (1LL << (bits - 1)))
			                                           : (v >= 0 && v < (1LL << bits));
			if (!ok) {
				b200_set_error("b200_filter_project: constant node %d holds %lld, outside its type %d", i, (long long)v,
				               nd.type);
				return B200_ERR_INVALID;
			}
		}
		if (nd.op == B200_EXPR_COLREF) {
			if (nd.col < 0 || nd.col >= (int)in->cols.size() || nd.col >= 256) {
				b200_set_error("b200_filter_project: node %d references column %d (batch has %d)", i, nd.col,
				               (int)in->cols.size());
				return B200_ERR_INVALID;
			}
			if (in->cols[nd.col].type != nd.type) {
				b200_set_error("b200_filter_project: node %d type %d does not match column type %d", i, nd.type,
				               in->cols[nd.col].type);
				return B200_ERR_INVALID;
			}
			if (col_map[nd.col] < 0) {
				if (nmapped >= MAX_PCOLS) {
					b200_set_error("b200_filter_project: at most %d distinct input columns", MAX_PCOLS);
					return B200_ERR_INVALID;
				}
				prog.cols[nmapped] = in->cols[nd.col];
				col_map[nd.col] = nmapped++;
			}
			prog.nodes[i].col = col_map[nd.col];
		}
	}
	for (int j = 0; j < nproj; j++) {
		if (proj_roots[j] < 0 || proj_roots[j] >= nnodes) {
			b200_set_error("b200_filter_project: projection root %d out of range", proj_roots[j]);
			return B200_ERR_INVALID;
		}
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	uint64_t n = in->nrows;
	*out_count = 0;
	if (out) {
		*out = nullptr;
	}
	uint64_t ntiles = (n + TILE_ROWS - 1) / TILE_ROWS;
	uint32_t *mask32 = (uint32_t *)out_mask;
	void *own_mask = nullptr;
	uint32_t *tile_counts = nullptr;
	uint64_t *tile_offsets = nullptr;
	int *flags = (int *)(ctx->dev_scratch + 8);
	uint64_t *total_dev = ctx->dev_scratch;
	CUDA_TRY(cudaMemsetAsync(ctx->dev_scratch, 0, 16 * sizeof(uint64_t), ctx->stream));
	uint64_t count = n;
	int grid = (int)(ntiles < (uint64_t)ctx->sm_count * 8 ? (ntiles ? ntiles : 1) : (uint64_t)ctx->sm_count * 8);
	// Single-pass path (filter_tile.cu): `col CMP const` AND-trees over flat non-NULL integer columns, projections =
	// plain column references.  The output columns are allocated for n rows (the survivor count is only known after
	// the one kernel) and trimmed afterwards; inputs beyond the budget below take the exactly-sized two-pass path.
	if (filter_root >= 0 && n > 0 && nproj > 0 && getenv("B200_FILTER_FUSED")) {
		size_t out_bytes = 0;
		bool plain = true;
		for (int j = 0; j < nproj; j++) {
			const b200_expr_node &nd = prog.nodes[proj_roots[j]];
			plain = plain && nd.op == B200_EXPR_COLREF && !prog.cols[nd.col].validity;
			out_bytes += (size_t)n * b200_type_size(nd.type);
		}
		if (plain && out_bytes <= ((size_t)24 << 30)) {
			b200_batch *fb = b200_batch_new(ctx, n);
			void *odata[MAX_PROJ];
			int rc = B200_OK;
			for (int j = 0; j < nproj && rc == B200_OK; j++) {
				rc = b200_batch_add_flat(fb, nodes[proj_roots[j]].type, n, false, &odata[j], nullptr);
			}
			uint32_t *status = nullptr;
			rc = rc ? rc : b200_dev_alloc(ctx, ntiles * 4 + 16, (void **)&status);
			if (rc == B200_OK) {
				CUDA_TRY(cudaMemsetAsync(status, 0, ntiles * 4, ctx->stream));
				if (out_mask) {
					CUDA_TRY(cudaMemsetAsync(out_mask + (n + 63) / 64 - 1, 0, 8, ctx->stream));
				}
				rc = b200_filter_fused_tile(ctx, prog.nodes, filter_root, proj_roots, nproj, odata, prog.cols, nmapped, n,
				                            (uint32_t *)out_mask, out_sel, status, (unsigned long long *)total_dev);
			}
			if (rc == B200_OK) {
				cudaError_t e = cudaMemcpyAsync(ctx->pinned_scratch, total_dev, 8, cudaMemcpyDeviceToHost, ctx->stream);
				e = e ? e : cudaStreamSynchronize(ctx->stream);
				e = e ? e : cudaGetLastError();
				b200_dev_free(ctx, status);
				if (e != cudaSuccess) {
					b200_batch_free(fb);
					return b200_cuda_fail(e, "filter_project(fused)", __FILE__, __LINE__);
				}
				ctx->d2h_bytes += 8;
				fb->nrows = ctx->pinned_scratch[0];
				*out_count = fb->nrows;
				*out = fb;
				return B200_OK;
			}
			b200_dev_free(ctx, status);
			b200_batch_free(fb);
			if (rc != B200_ERR_INVALID) {
				return rc;
			}
		}
	}
	if (filter_root >= 0 && n > 0) {
		if (!mask32) {
			B200_TRY(b200_dev_alloc(ctx, ((n + 63) / 64) * 8 + 16, &own_mask));
			mask32 = (uint32_t *)own_mask;
		}
		// zero the tail word so that bits past n are 0
		CUDA_TRY(cudaMemsetAsync((uint64_t *)mask32 + (n + 63) / 64 - 1, 0, 8, ctx->stream));
		B200_TRY(b200_dev_alloc(ctx, ntiles * 4 + 16, (void **)&tile_counts));
		B200_TRY(b200_dev_alloc(ctx, (ntiles + 4 + (ntiles + SCAN_CHUNK - 1) / SCAN_CHUNK) * 8 + 16, (void **)&tile_offsets));
		int trc = b200_filter_mask_tile(ctx, prog.nodes, filter_root, prog.cols, nmapped, n, mask32, tile_counts);
		if (trc == B200_ERR_INVALID) {
			filter_mask_kernel<<<grid, 256, 0, ctx->stream>>>(prog, filter_root, closure_of(prog, 1u << filter_root), n,
			                                                  mask32, tile_counts, flags);
			ctx->launches++;
		} else if (trc != B200_OK) {
			b200_dev_free(ctx, own_mask);
			b200_dev_free(ctx, tile_counts);
			b200_dev_free(ctx, tile_offsets);
			return trc;
		}
		{
			uint64_t nchunks = (ntiles + SCAN_CHUNK - 1) / SCAN_CHUNK;
			uint64_t *chunk_totals = tile_offsets + ntiles + 2; // tail of the same allocation
			tile_scan_local_kernel<<<(unsigned)nchunks, 1024, 0, ctx->stream>>>(tile_counts, tile_offsets, ntiles,
			                                                                    chunk_totals);
			tile_scan_chunks_kernel<<<1, 32, 0, ctx->stream>>>(chunk_totals, nchunks, total_dev);
			tile_scan_add_kernel<<<(unsigned)nchunks, 1024, 0, ctx->stream>>>(tile_offsets, ntiles, chunk_totals);
			ctx->launches += 3;
		}
		CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch, total_dev, 8, cudaMemcpyDeviceToHost, ctx->stream));
		CUDA_TRY(cudaStreamSynchronize(ctx->stream));
		ctx->d2h_bytes += 8;
		count = ctx->pinned_scratch[0];
	}
	b200_batch *ob = nullptr;
	ProjOut po;
	po.n = nproj;
	if (nproj > 0) {
		ob = b200_batch_new(ctx, count);
		std::vector<int> memo(nnodes, -1);
		for (int j = 0; j < nproj; j++) {
			int r = proj_roots[j];
			bool nullable = node_may_be_null(prog, r, memo);
			void *d;
			uint64_t *v;
			int rc = b200_batch_add_flat(ob, nodes[r].type, count, nullable, &d, &v);
			if (rc != B200_OK) {
				b200_batch_free(ob);
				return rc;
			}
			po.data[j] = d;
			po.validity[j] = v;
			po.root[j] = r;
			po.type[j] = nodes[r].type;
			if (v && count) {
				uint64_t words = (count + 63) / 64;
				fill_u64_kernel2<<<grid_for(words, 256, 1, 1024), 256, 0, ctx->stream>>>(v, words, ~0ULL);
				ctx->launches++;
			}
		}
	}
	if (n > 0 && count > 0 && (nproj > 0 || out_sel)) {
		uint32_t proots = 0;
		for (int j = 0; j < nproj; j++) {
			proots |= 1u << proj_roots[j];
		}
		uint32_t pneed = closure_of(prog, proots);
		int trc = B200_ERR_INVALID;
		if (filter_root >= 0 && nproj > 0) {
			bool nullable_out = false;
			for (int j = 0; j < nproj; j++) {
				nullable_out = nullable_out || po.validity[j] != nullptr;
			}
			if (!nullable_out) {
				trc = b200_filter_compact_tile(ctx, prog.nodes, proj_roots, nproj, po.data, prog.cols, nmapped, n, mask32,
				                               tile_offsets, out_sel);
			}
		}
		if (trc == B200_OK) {
			ctx->launches--; // counted by the tile launcher; keep the increment below balanced
		} else if (trc != B200_ERR_INVALID) {
			b200_batch_free(ob);
			b200_dev_free(ctx, own_mask);
			b200_dev_free(ctx, tile_counts);
			b200_dev_free(ctx, tile_offsets);
			return trc;
		} else if (filter_root >= 0) {
			compact_kernel<false>
			    <<<grid, 256, 0, ctx->stream>>>(prog, po, pneed, n, mask32, tile_offsets, out_sel, flags);
		} else {
			compact_kernel<true><<<grid, 256, 0, ctx->stream>>>(prog, po, pneed, n, nullptr, nullptr, out_sel, flags);
		}
		ctx->launches++;
	}
	CUDA_TRY(cudaMemcpyAsync(ctx->pinned_scratch + 8, flags, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
	cudaError_t e = cudaStreamSynchronize(ctx->stream);
	if (e == cudaSuccess) {
		e = cudaGetLastError();
	}
	b200_dev_free(ctx, own_mask);
	b200_dev_free(ctx, tile_counts);
	b200_dev_free(ctx, tile_offsets);
	if (e != cudaSuccess) {
		b200_batch_free(ob);
		return b200_cuda_fail(e, "filter_project", __FILE__, __LINE__);
	}
	if (*(int *)(ctx->pinned_scratch + 8)) {
		b200_batch_free(ob);
		b200_set_error("Overflow in integer/DECIMAL arithmetic of a projected expression");
		return B200_ERR_OVERFLOW;
	}
	*out_count = count;
	if (out) {
		*out = ob;
	}
	return B200_OK;
}
