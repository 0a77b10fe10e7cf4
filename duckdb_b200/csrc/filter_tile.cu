// K5 filter_select + project, TMA-staged fast path.
//
// Eligibility (checked on the host, everything else takes the generic interpreter in filter.cu):
//   predicate  = AND of <= 6 terms  `column CMP constant`  over FLAT integer / date columns without NULLs
//   projection = plain references to FLAT columns without NULLs
// which covers the scan-side filters of the BASELINE configs (l_shipdate < DATE, date ranges of Q14/Q3/Q6).
// Two kernels share the 2048-row tiling and the mask / tile-count layout of filter.cu:
//   A' filter_mask_tile_kernel   stage predicate columns by TMA, evaluate, ballot -> mask words + tile counts
//   C' compact_tile_kernel       stage projected columns by TMA, ordered compaction of the surviving rows
// (the tile-count scan in between is filter.cu's tile_scan_kernel).
#include "common.cuh"
#include "tile_pipe.cuh"
#include <cstring>
#include <cstdlib>

#define FT_THREADS 256
#define FT_TILE 2048
#define FT_MAX_TERMS 6
#define FT_MAX_PROJ 12
#define FT_STAGES 3

struct FilterTerm {
	int col;       // tile column index
	int width;     // bytes
	int is_signed;
	int op;        // b200_expr_op comparison
	int64_t value; // constant (sign- or zero-extended)
	// the same predicate as a wrap-around range test in the column's own width (valid when the constant is
	// representable there): row passes  <=>  ((T)(v - lo) <= span) != neg
	uint64_t lo, span;
	int neg;
};

struct MaskArgs {
	TileCols tc;
	FilterTerm t[FT_MAX_TERMS];
	int nterms;
	int lean; // every constant is representable in its column's type: compare in the native width
	uint64_t n;
	uint32_t *mask32;
	uint32_t *tile_counts;
	int stages;
};

struct CompactArgs {
	TileCols tc;
	int nproj;
	int col[FT_MAX_PROJ];
	int width[FT_MAX_PROJ];
	void *out[FT_MAX_PROJ];
	uint64_t n;
	const uint32_t *mask32;
	const uint64_t *tile_offsets;
	uint32_t *out_sel;
	int stages;
};

#define FT_ROWS (FT_TILE / FT_THREADS)

// keep[k] &= (value(row k) CMP constant) for the thread's FT_ROWS rows of the tile.  The width / signedness / op
// dispatch happens ONCE per term (outside the row loop); the comparison itself is branch-free:
// keep = (lt & want_lt) | (eq & want_eq) | (gt & want_gt).
template <class T>
__device__ __forceinline__ void eval_term_rows(const unsigned char *col, int tid, uint32_t rows_in_tile, int64_t value,
                                               bool unsigned64, uint32_t want, bool (&keep)[FT_ROWS]) {
	const T *p = (const T *)col;
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		uint32_t r = k * FT_THREADS + tid;
		if (r < rows_in_tile) {
			int64_t v = (int64_t)p[r];
			bool lt = unsigned64 ? ((uint64_t)v < (uint64_t)value) : (v < value);
			bool eq = v == value;
			uint32_t bits = lt ? 1u : (eq ? 2u : 4u);
			keep[k] = keep[k] && (bits & want);
		} else {
			keep[k] = false;
		}
	}
}

// Lean evaluation of one `column CMP constant` term on a FULL 2048-row (sub-)tile: the comparison runs in the column's
// own width (one ISETP for <= 4-byte types) and the operator is resolved once per term, not per row.  (A per-row
// operator / width dispatch makes the kernel issue-bound on a 4-byte column.)
template <class T, class CMP>
__device__ __forceinline__ void eval_rows_lean(const T *p, int tid, T value, bool (&keep)[FT_ROWS], CMP cmp) {
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		keep[k] = keep[k] && cmp(p[k * FT_THREADS + tid], value);
	}
}

template <class T>
__device__ __forceinline__ void eval_term_lean(const unsigned char *col, int tid, int64_t value64, int op, bool (&keep)[FT_ROWS]) {
	const T *p = (const T *)col;
	// a constant outside T's range cannot be compared in T: the caller routes those terms to the generic path
	const T value = (T)value64;
	switch (op) {
	case B200_EXPR_EQ:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a == b; });
		break;
	case B200_EXPR_NE:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a != b; });
		break;
	case B200_EXPR_LT:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a < b; });
		break;
	case B200_EXPR_LE:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a <= b; });
		break;
	case B200_EXPR_GT:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a > b; });
		break;
	default:
		eval_rows_lean<T>(p, tid, value, keep, [](T a, T b) { return a >= b; });
		break;
	}
}

// Range form of a term on a full 2048-row sub-tile: ONE subtract and ONE unsigned compare per row whatever the operator
// (LT / LE / GT / GE / EQ are ranges [lo, hi] of the type's value order, NE the complement; (T)(v - lo) <= (T)(hi - lo)
// in wrap-around arithmetic of the column's width holds exactly for lo <= v <= hi, signed or unsigned).  Returns bit k
// = row k * FT_THREADS + tid passes.  (A switch per operator makes the kernel
// issue-bound on a 4-byte column.)
template <class T>
__device__ __forceinline__ uint32_t range_bits(const unsigned char *col, int tid, uint64_t lo64, uint64_t span64, int neg) {
	const T *p = (const T *)col;
	const T lo = (T)lo64, span = (T)span64;
	uint32_t b = 0;
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		T d = (T)(p[k * FT_THREADS + tid] - lo);
		b |= (uint32_t)(d <= span) << k;
	}
	return neg ? ~b : b;
}

__device__ __forceinline__ uint32_t eval_terms_range(const FilterTerm *terms, int nterms, const TileCols &tc,
                                                     const unsigned char *stage, size_t row_off, int tid) {
	uint32_t bits = (1u << FT_ROWS) - 1;
#pragma unroll 1
	for (int i = 0; i < nterms; i++) {
		const FilterTerm &t = terms[i];
		const unsigned char *col = stage + tc.c[t.col].smem_off + row_off * t.width;
		switch (t.width) {
		case 1:
			bits &= range_bits<uint8_t>(col, tid, t.lo, t.span, t.neg);
			break;
		case 2:
			bits &= range_bits<uint16_t>(col, tid, t.lo, t.span, t.neg);
			break;
		case 4:
			bits &= range_bits<uint32_t>(col, tid, t.lo, t.span, t.neg);
			break;
		default:
			bits &= range_bits<uint64_t>(col, tid, t.lo, t.span, t.neg);
			break;
		}
	}
	return bits;
}

// all terms of a predicate on a full (sub-)tile; `lean_ok` per term is decided on the host (constant representable in
// the column type)
__device__ __forceinline__ void eval_terms_full(const FilterTerm *terms, int nterms, const TileCols &tc, const unsigned char *stage,
                                                size_t row_off, int tid, bool (&keep)[FT_ROWS]) {
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		keep[k] = true;
	}
#pragma unroll 1
	for (int i = 0; i < nterms; i++) {
		const FilterTerm &t = terms[i];
		const unsigned char *col = stage + tc.c[t.col].smem_off + row_off * t.width;
		switch (t.width * 2 + (t.is_signed ? 1 : 0)) {
		case 2:
			eval_term_lean<uint8_t>(col, tid, t.value, t.op, keep);
			break;
		case 3:
			eval_term_lean<int8_t>(col, tid, t.value, t.op, keep);
			break;
		case 4:
			eval_term_lean<uint16_t>(col, tid, t.value, t.op, keep);
			break;
		case 5:
			eval_term_lean<int16_t>(col, tid, t.value, t.op, keep);
			break;
		case 8:
			eval_term_lean<uint32_t>(col, tid, t.value, t.op, keep);
			break;
		case 9:
			eval_term_lean<int32_t>(col, tid, t.value, t.op, keep);
			break;
		case 16:
			eval_term_lean<uint64_t>(col, tid, t.value, t.op, keep);
			break;
		default:
			eval_term_lean<int64_t>(col, tid, t.value, t.op, keep);
			break;
		}
	}
}

__device__ __forceinline__ uint32_t want_bits(int op) {
	switch (op) {
	case B200_EXPR_EQ:
		return 2u;
	case B200_EXPR_NE:
		return 5u;
	case B200_EXPR_LT:
		return 1u;
	case B200_EXPR_LE:
		return 3u;
	case B200_EXPR_GT:
		return 4u;
	default:
		return 6u; // GE
	}
}

// ONE range term over a FULL super-tile: compare -> ballot -> mask word / count, nothing else in the loop (the width
// dispatch, the column pointer and the term's constants sit outside).  ~8 instructions per row.
template <class T, int NSUB>
__device__ __forceinline__ void mask_single_term(const unsigned char *col, uint64_t lo64, uint64_t span64, int neg,
                                                 uint32_t *mask_words, uint32_t (&warp_cnt)[NSUB][FT_THREADS / 32], int tid) {
	const T *p = (const T *)col + tid;
	const T lo = (T)lo64, span = (T)span64;
	const uint32_t flip = neg ? 0xffffffffu : 0u;
	const int lane = tid & 31, warp = tid >> 5;
	uint32_t *mrow = mask_words + warp;
#pragma unroll
	for (int sub = 0; sub < NSUB; sub++) {
		uint32_t cnt = 0;
#pragma unroll
		for (int k = 0; k < FT_ROWS; k++) {
			const T d = (T)(p[sub * FT_TILE + k * FT_THREADS] - lo);
			const uint32_t m = __ballot_sync(0xffffffffu, d <= span) ^ flip;
			if (lane == 0) {
				mrow[sub * (FT_TILE / 32) + k * (FT_THREADS / 32)] = m;
			}
			cnt += __popc(m);
		}
		if (lane == 0) {
			warp_cnt[sub][warp] = cnt;
		}
	}
}

// A' (two-pass path).  The predicate columns are narrow (a DATE is 4 bytes): a 2048-row tile of one column is 8 KB
// and the per-tile costs (TMA issue by one thread, mbarrier wait, barriers) dominate.  The mask kernel therefore stages SUPER-tiles of MROWS x 512 rows (up to 16 K rows) and walks them in
// 2048-row sub-tiles, so that the mask words and the per-2048-row counts keep the layout the scan / compaction expect.
template <int MROWS>
__global__ void __launch_bounds__(FT_THREADS) filter_mask_tile_kernel(const __grid_constant__ MaskArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * FT_STAGES];
	constexpr int NSUB = MROWS / FT_ROWS; // 2048-row sub-tiles per super-tile
	__shared__ uint32_t warp_cnt[NSUB][FT_THREADS / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	// config 1's shape - one `col CMP const` term - has its own loop over the whole super-tile
	const bool single = A.lean && A.nterms == 1;
	const FilterTerm &t0 = A.t[0];
	const uint32_t col0 = A.tc.c[t0.col].smem_off;
	tp_tile_loop_sync(A.tc, A.stages, smem_raw, bars, 0, A.n, [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		if (single && rows_in_tile == (uint32_t)MROWS * FT_THREADS) {
			uint32_t *words = A.mask32 + (row0 >> 5);
			switch (t0.width) {
			case 1:
				mask_single_term<uint8_t, NSUB>(stage + col0, t0.lo, t0.span, t0.neg, words, warp_cnt, tid);
				break;
			case 2:
				mask_single_term<uint16_t, NSUB>(stage + col0, t0.lo, t0.span, t0.neg, words, warp_cnt, tid);
				break;
			case 4:
				mask_single_term<uint32_t, NSUB>(stage + col0, t0.lo, t0.span, t0.neg, words, warp_cnt, tid);
				break;
			default:
				mask_single_term<uint64_t, NSUB>(stage + col0, t0.lo, t0.span, t0.neg, words, warp_cnt, tid);
				break;
			}
		} else {
#pragma unroll 1
		for (int sub = 0; sub < NSUB; sub++) {
			const uint32_t sub_row = (uint32_t)sub * FT_TILE;
			const uint32_t rows = rows_in_tile > sub_row ? (rows_in_tile - sub_row < FT_TILE ? rows_in_tile - sub_row : FT_TILE) : 0;
			bool keep[FT_ROWS];
			uint32_t cnt = 0;
			if (rows == FT_TILE && A.lean) {
				// full sub-tile: lean compares, mask words through one running pointer
				const uint32_t bits = eval_terms_range(A.t, A.nterms, A.tc, stage, sub_row, tid);
				uint32_t *mrow = A.mask32 + ((row0 + sub_row) >> 5) + warp;
#pragma unroll
				for (int k = 0; k < FT_ROWS; k++) {
					uint32_t m = __ballot_sync(0xffffffffu, (bits >> k) & 1u);
					if (lane == 0) {
						mrow[k * (FT_THREADS / 32)] = m;
					}
					cnt += __popc(m);
				}
			} else {
#pragma unroll
				for (int k = 0; k < FT_ROWS; k++) {
					keep[k] = true;
				}
#pragma unroll 1
				for (int i = 0; i < A.nterms; i++) {
					const FilterTerm &t = A.t[i];
					const unsigned char *col = stage + A.tc.c[t.col].smem_off + (size_t)sub_row * t.width;
					uint32_t want = want_bits(t.op);
					switch (t.width * 2 + (t.is_signed ? 1 : 0)) {
					case 2:
						eval_term_rows<uint8_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 3:
						eval_term_rows<int8_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 4:
						eval_term_rows<uint16_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 5:
						eval_term_rows<int16_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 8:
						eval_term_rows<uint32_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 9:
						eval_term_rows<int32_t>(col, tid, rows, t.value, false, want, keep);
						break;
					case 16:
						eval_term_rows<uint64_t>(col, tid, rows, t.value, true, want, keep);
						break;
					default:
						eval_term_rows<int64_t>(col, tid, rows, t.value, false, want, keep);
						break;
					}
				}
#pragma unroll
				for (int k = 0; k < FT_ROWS; k++) {
					uint32_t m = __ballot_sync(0xffffffffu, keep[k]);
					uint32_t group_row = k * FT_THREADS + warp * 32;
					if (lane == 0 && group_row < rows) {
						A.mask32[((row0 + sub_row) >> 5) + (group_row >> 5)] = m;
					}
					cnt += __popc(m);
				}
			}
			if (lane == 0) {
				warp_cnt[sub][warp] = cnt;
			}
		}
		}
		__syncthreads();
		if (tid < NSUB && (uint32_t)tid * FT_TILE < rows_in_tile) {
			uint32_t t = 0;
			for (int w = 0; w < FT_THREADS / 32; w++) {
				t += warp_cnt[tid][w];
			}
			A.tile_counts[row0 / FT_TILE + tid] = t;
		}
	});
}

// copy column values of the selected rows: the width dispatch is outside the row loop
template <class T>
__device__ __forceinline__ void copy_rows(void *out, const unsigned char *col, const uint32_t (&r)[FT_ROWS],
                                          const uint64_t (&opos)[FT_ROWS], const bool (&sel)[FT_ROWS]) {
	const T *p = (const T *)col;
	T *o = (T *)out;
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		if (sel[k]) {
			o[opos[k]] = p[r[k]];
		}
	}
}

__global__ void __launch_bounds__(FT_THREADS) compact_tile_kernel(const __grid_constant__ CompactArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[2 * FT_STAGES];
	__shared__ uint32_t group_mask[FT_TILE / 32];
	__shared__ uint32_t group_base[FT_TILE / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	tp_tile_loop_sync(A.tc, A.stages, smem_raw, bars, 0, A.n, [&](const unsigned char *stage, uint64_t row0, uint32_t rows_in_tile) {
		const uint64_t out0 = A.tile_offsets[row0 / FT_TILE];
		// the tile's 64 mask words and their exclusive prefix (two warps)
		if (tid < FT_TILE / 32) {
			uint32_t m = (uint32_t)tid * 32 < rows_in_tile ? A.mask32[(row0 >> 5) + tid] : 0;
			group_mask[tid] = m;
			uint32_t c = __popc(m), incl = c;
#pragma unroll
			for (int off = 1; off < 32; off <<= 1) {
				uint32_t t = __shfl_up_sync(0xffffffffu, incl, off);
				if (lane >= off) {
					incl += t;
				}
			}
			group_base[tid] = incl - c;
		}
		__syncthreads();
		if (tid >= 32 && tid < 64) {
			group_base[tid] += group_base[31] + __popc(group_mask[31]);
		}
		__syncthreads();
		uint32_t r[FT_ROWS];
		uint64_t opos[FT_ROWS];
		bool sel[FT_ROWS];
#pragma unroll
		for (int k = 0; k < FT_ROWS; k++) {
			int g = k * (FT_THREADS / 32) + warp; // rows g*32 .. g*32+31
			uint32_t m = group_mask[g];
			sel[k] = (m >> lane) & 1;
			r[k] = g * 32 + lane;
			opos[k] = out0 + group_base[g] + __popc(m & ((1u << lane) - 1));
			if (sel[k] && A.out_sel) {
				A.out_sel[opos[k]] = (uint32_t)(row0 + r[k]);
			}
		}
#pragma unroll 1
		for (int j = 0; j < A.nproj; j++) {
			const unsigned char *col = stage + A.tc.c[A.col[j]].smem_off;
			switch (A.width[j]) {
			case 1:
				copy_rows<uint8_t>(A.out[j], col, r, opos, sel);
				break;
			case 2:
				copy_rows<uint16_t>(A.out[j], col, r, opos, sel);
				break;
			case 4:
				copy_rows<uint32_t>(A.out[j], col, r, opos, sel);
				break;
			default:
				copy_rows<uint64_t>(A.out[j], col, r, opos, sel);
				break;
			}
		}
	});
}

// ---------------------------------------------------------------------------------------------------------------
// Single-pass filter + projection: ONE kernel evaluates the predicate on the staged tile, orders the tiles' outputs,
// compacts the surviving values of every projected column in shared memory and writes them out as one contiguous run
// per tile (full 128-byte lines, whatever the selectivity).  Every input byte is read once.
// Output order without a serial chain: tiles are assigned round-robin to G co-resident CTAs, every tile publishes its
// survivor count in a status word as soon as it has evaluated the predicate, and
//     excl(t) = excl(t - G) + sum of the counts of tiles t-G .. t-1
// where excl(t - G) is the value the SAME CTA computed one iteration earlier (kept in a register).  The G counts are
// read by the whole CTA in one batch of parallel loads - a wait on publication only, never on another tile's prefix.
// (A first version used the classic chained look-back: at 2048-row tiles the chain advances ~32 tiles per L2 round
// trip, far fewer than HBM delivers, and the CTAs park at the barrier behind one spinning thread.)
#define FF_PUBLISHED 0x80000000u

struct FusedArgs {
	TileCols tc;
	FilterTerm t[FT_MAX_TERMS];
	int nterms;
	int lean;
	int nproj;
	int col[FT_MAX_PROJ];
	int width[FT_MAX_PROJ];
	uint32_t cbuf_off[FT_MAX_PROJ]; // byte offset of column j's compaction buffer (FT_TILE values) after the stages
	void *out[FT_MAX_PROJ];
	uint64_t n;
	uint32_t *mask32;        // optional
	uint32_t *out_sel;       // optional (compacted through the buffer at sel_off)
	uint32_t sel_off;
	uint32_t *status;           // one word per tile (count | FF_PUBLISHED), zeroed before the launch
	unsigned long long *total;  // survivors (written by the CTA of the last tile)
	int stages;
};

template <class T>
__device__ __forceinline__ void stage_selected(unsigned char *cbuf, const unsigned char *col, int tid,
                                               const uint32_t (&lpos)[FT_ROWS], const bool (&keep)[FT_ROWS]) {
	const T *p = (const T *)col;
	T *o = (T *)cbuf;
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		if (keep[k]) {
			o[lpos[k]] = p[k * FT_THREADS + tid];
		}
	}
}

template <class T>
__device__ __forceinline__ void copy_run(void *out, uint64_t out0, const unsigned char *cbuf, uint32_t count, int tid) {
	const T *c = (const T *)cbuf;
	T *o = (T *)out + out0;
	for (uint32_t i = tid; i < count; i += FT_THREADS) {
		o[i] = c[i];
	}
}

// evaluate the predicate terms on the thread's FT_ROWS rows of a staged tile
__device__ __forceinline__ void ff_eval_terms(const FusedArgs &A, const unsigned char *stage, int tid, uint32_t rows_in_tile,
                                              bool (&keep)[FT_ROWS]) {
#pragma unroll
	for (int k = 0; k < FT_ROWS; k++) {
		keep[k] = true;
	}
#pragma unroll 1
	for (int i = 0; i < A.nterms; i++) {
		const FilterTerm &ft = A.t[i];
		const unsigned char *col = stage + A.tc.c[ft.col].smem_off;
		uint32_t want = want_bits(ft.op);
		switch (ft.width * 2 + (ft.is_signed ? 1 : 0)) {
		case 2:
			eval_term_rows<uint8_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 3:
			eval_term_rows<int8_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 4:
			eval_term_rows<uint16_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 5:
			eval_term_rows<int16_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 8:
			eval_term_rows<uint32_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 9:
			eval_term_rows<int32_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		case 16:
			eval_term_rows<uint64_t>(col, tid, rows_in_tile, ft.value, true, want, keep);
			break;
		default:
			eval_term_rows<int64_t>(col, tid, rows_in_tile, ft.value, false, want, keep);
			break;
		}
	}
}

// Software-pipelined over the CTA's tiles: iteration k evaluates tile k and publishes its count (phase A), then
// compacts tile k-1 (phase B), whose prefix needs the counts other CTAs published one phase A ago - by now they are
// visible, so nobody spins.  (Without the skew every CTA waits every tile for the slowest publication of its round.)  Tile k-1's stage and mask stay alive
// until its phase B is done; the ring therefore holds S >= 3 stages and refills the stage of tile k-1 with tile
// k-1+S at the end of iteration k.
__global__ void __launch_bounds__(FT_THREADS) filter_fused_tile_kernel(const __grid_constant__ FusedArgs A) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ uint64_t bars[4];
	__shared__ uint32_t gmask[2][FT_TILE / 32];
	__shared__ uint32_t gbase[2][FT_TILE / 32 + 1];
	__shared__ uint32_t warp_part[FT_THREADS / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int S = A.stages;
	unsigned char *cbufs = smem_raw + (size_t)S * A.tc.stage_bytes;
	const uint64_t G = gridDim.x;
	const uint64_t ntiles = (A.n + FT_TILE - 1) / FT_TILE, nfull = A.n / FT_TILE;
	const uint64_t nk = blockIdx.x < ntiles ? (ntiles - blockIdx.x + G - 1) / G : 0; // tiles of this CTA
	if (tid == 0) {
		for (int s = 0; s < S; s++) {
			tp_mbar_init(&bars[s], 1);
		}
		tp_fence_mbar_init();
	}
	__syncthreads();
	if (tid == 0) {
		for (uint64_t j = 0; j < (uint64_t)S && j < nk; j++) {
			uint64_t t = blockIdx.x + j * G;
			if (t < nfull) {
				tp_issue_full(A.tc, smem_raw + (size_t)j * A.tc.stage_bytes, &bars[j], t * FT_TILE);
			}
		}
	}
	uint64_t carry = 0; // exclusive prefix of the tile compacted last
	for (uint64_t k = 0; k <= nk; k++) {
		// ---- the counts of the G tiles before tile k-1 (all earlier tiles when it is the CTA's first): the loads are issued
		// FIRST, their L2 latency is covered by the predicate evaluation of tile k below
		constexpr int WPT = 4; // window words per thread held in registers (grids beyond WPT * FT_THREADS tiles loop)
		uint32_t wv[WPT];
		uint64_t wbase = 0, wend = 0;
		if (k >= 1) {
			const uint64_t tp = blockIdx.x + (k - 1) * G;
			wbase = tp >= G ? tp - G : 0;
			wend = tp;
#pragma unroll
			for (int q = 0; q < WPT; q++) {
				uint64_t i = wbase + tid + (uint64_t)q * FT_THREADS;
				wv[q] = i < wend ? *(volatile uint32_t *)&A.status[i] : FF_PUBLISHED;
			}
		}
		// ---- phase A(k): predicate, mask words, (count published after the barrier)
		if (k < nk) {
			const uint64_t t = blockIdx.x + k * G;
			const int s = (int)(k % S);
			unsigned char *stage = smem_raw + (size_t)s * A.tc.stage_bytes;
			uint32_t rows_in_tile = FT_TILE;
			if (t < nfull) {
				tp_wait(&bars[s], (uint32_t)((k / S) & 1));
			} else {
				rows_in_tile = (uint32_t)(A.n - t * FT_TILE);
				tp_copy_ragged(A.tc, stage, t * FT_TILE, rows_in_tile);
				__syncthreads();
			}
			bool keep[FT_ROWS];
			if (rows_in_tile == FT_TILE && A.lean) {
				eval_terms_full(A.t, A.nterms, A.tc, stage, 0, tid, keep);
			} else {
				ff_eval_terms(A, stage, tid, rows_in_tile, keep);
			}
#pragma unroll
			for (int j = 0; j < FT_ROWS; j++) {
				uint32_t m = __ballot_sync(0xffffffffu, keep[j]);
				int g = j * (FT_THREADS / 32) + warp;
				if (lane == 0) {
					gmask[k & 1][g] = m;
					if (A.mask32 && (uint32_t)g * 32 < rows_in_tile) {
						A.mask32[(t * FT_TILE >> 5) + g] = m;
					}
				}
			}
		}
		if (k >= 1) {
			uint32_t part = 0;
#pragma unroll
			for (int q = 0; q < WPT; q++) {
				uint64_t i = wbase + tid + (uint64_t)q * FT_THREADS;
				while (!(wv[q] & FF_PUBLISHED)) { // (rare) not yet published when it was prefetched
					wv[q] = *(volatile uint32_t *)&A.status[i];
				}
				part += wv[q] & ~FF_PUBLISHED;
			}
			for (uint64_t i = wbase + tid + (uint64_t)WPT * FT_THREADS; i < wend; i += FT_THREADS) {
				uint32_t v;
				do {
					v = *(volatile uint32_t *)&A.status[i];
				} while (!(v & FF_PUBLISHED));
				part += v & ~FF_PUBLISHED;
			}
#pragma unroll
			for (int off = 16; off; off >>= 1) {
				part += __shfl_xor_sync(0xffffffffu, part, off);
			}
			if (lane == 0) {
				warp_part[warp] = part;
			}
		}
		__syncthreads();
		if (k < nk && warp == 0) {
			// exclusive prefix over the 64 group counts of tile k (two per lane); lane 31 publishes the tile total
			uint32_t a = __popc(gmask[k & 1][2 * lane]), b = __popc(gmask[k & 1][2 * lane + 1]);
			uint32_t sum = a + b, incl = sum;
#pragma unroll
			for (int off = 1; off < 32; off <<= 1) {
				uint32_t v = __shfl_up_sync(0xffffffffu, incl, off);
				if (lane >= off) {
					incl += v;
				}
			}
			gbase[k & 1][2 * lane] = incl - sum;
			gbase[k & 1][2 * lane + 1] = incl - sum + a;
			if (lane == 31) {
				gbase[k & 1][FT_TILE / 32] = incl;
				*(volatile uint32_t *)&A.status[blockIdx.x + k * G] = FF_PUBLISHED | incl;
			}
		}
		// ---- phase B(k-1): ordered compaction of tile k-1
		if (k >= 1) {
			const uint64_t tp = blockIdx.x + (k - 1) * G;
			const int pb = (int)((k - 1) & 1);
			const unsigned char *stage = smem_raw + (size_t)((k - 1) % S) * A.tc.stage_bytes;
			uint32_t window = 0;
#pragma unroll
			for (int w = 0; w < FT_THREADS / 32; w++) {
				window += warp_part[w];
			}
			carry += window; // = exclusive prefix of tile k-1 (identical in every thread)
			const uint64_t out0 = carry;
			const uint32_t total = gbase[pb][FT_TILE / 32]; // written by warp 0 one iteration ago
			if (tid == 0 && tp + 1 == ntiles) {
				*A.total = carry + total;
			}
			bool keep[FT_ROWS];
			uint32_t lpos[FT_ROWS];
#pragma unroll
			for (int j = 0; j < FT_ROWS; j++) {
				int g = j * (FT_THREADS / 32) + warp;
				uint32_t m = gmask[pb][g];
				keep[j] = (m >> lane) & 1;
				lpos[j] = gbase[pb][g] + __popc(m & ((1u << lane) - 1));
			}
			// compaction through shared memory: every column has its own buffer, so one barrier serves all of them
#pragma unroll 1
			for (int j = 0; j < A.nproj; j++) {
				const unsigned char *col = stage + A.tc.c[A.col[j]].smem_off;
				unsigned char *cb = cbufs + A.cbuf_off[j];
				switch (A.width[j]) {
				case 1:
					stage_selected<uint8_t>(cb, col, tid, lpos, keep);
					break;
				case 2:
					stage_selected<uint16_t>(cb, col, tid, lpos, keep);
					break;
				case 4:
					stage_selected<uint32_t>(cb, col, tid, lpos, keep);
					break;
				default:
					stage_selected<uint64_t>(cb, col, tid, lpos, keep);
					break;
				}
			}
			if (A.out_sel) {
				uint32_t *sb = (uint32_t *)(cbufs + A.sel_off);
#pragma unroll
				for (int j = 0; j < FT_ROWS; j++) {
					if (keep[j]) {
						sb[lpos[j]] = (uint32_t)(tp * FT_TILE + j * FT_THREADS + tid);
					}
				}
			}
			__syncthreads();
#pragma unroll 1
			for (int j = 0; j < A.nproj; j++) {
				const unsigned char *cb = cbufs + A.cbuf_off[j];
				switch (A.width[j]) {
				case 1:
					copy_run<uint8_t>(A.out[j], out0, cb, total, tid);
					break;
				case 2:
					copy_run<uint16_t>(A.out[j], out0, cb, total, tid);
					break;
				case 4:
					copy_run<uint32_t>(A.out[j], out0, cb, total, tid);
					break;
				default:
					copy_run<uint64_t>(A.out[j], out0, cb, total, tid);
					break;
				}
			}
			if (A.out_sel) {
				copy_run<uint32_t>(A.out_sel, out0, cbufs + A.sel_off, total, tid);
			}
		}
		__syncthreads(); // the compaction buffers and the stage of tile k-1 are free
		if (tid == 0 && k >= 1) {
			uint64_t kn = k - 1 + S;
			uint64_t t = blockIdx.x + kn * G;
			if (kn < nk && t < nfull) {
				int sn = (int)(kn % S);
				tp_issue_full(A.tc, smem_raw + (size_t)sn * A.tc.stage_bytes, &bars[sn], t * FT_TILE);
			}
		}
	}
}

static int ft_add_col(TileCols *tc, const void *ptr, uint32_t width) {
	for (int i = 0; i < tc->n; i++) {
		if (tc->c[i].ptr == (const unsigned char *)ptr && tc->c[i].width == width) {
			return i;
		}
	}
	if (tc->n >= TP_MAX_COLS) {
		return -1;
	}
	tc->c[tc->n].ptr = (const unsigned char *)ptr;
	tc->c[tc->n].width = width;
	return tc->n++;
}

static bool ft_col_ok(const DCol &c) {
	return c.vtype == B200_FLAT_VECTOR && !c.validity && tile_ptr_ok(c.data) && b200_type_is_integer(c.type);
}

// Collect `col CMP const` terms of an AND tree.  Returns false when the predicate has any other shape.
static bool collect_terms(const b200_expr_node *nodes, int root, const DCol *cols, int ncols, MaskArgs *A) {
	const b200_expr_node &nd = nodes[root];
	if (nd.op == B200_EXPR_AND) {
		return collect_terms(nodes, nd.left, cols, ncols, A) && collect_terms(nodes, nd.right, cols, ncols, A);
	}
	if (nd.op < B200_EXPR_EQ || nd.op > B200_EXPR_GE) {
		return false;
	}
	int l = nd.left, r = nd.right, op = nd.op;
	if (nodes[l].op == B200_EXPR_CONST && nodes[r].op == B200_EXPR_COLREF) {
		// const CMP col  ->  col CMP' const
		int t = l;
		l = r;
		r = t;
		op = op == B200_EXPR_LT ? B200_EXPR_GT : op == B200_EXPR_GT ? B200_EXPR_LT : op == B200_EXPR_LE ? B200_EXPR_GE
		     : op == B200_EXPR_GE ? B200_EXPR_LE : op;
	}
	if (nodes[l].op != B200_EXPR_COLREF || nodes[r].op != B200_EXPR_CONST || nodes[r].is_null) {
		return false;
	}
	int c = nodes[l].col;
	if (c < 0 || c >= ncols || !ft_col_ok(cols[c]) || A->nterms >= FT_MAX_TERMS) {
		return false;
	}
	FilterTerm &t = A->t[A->nterms];
	t.width = b200_type_size(cols[c].type);
	t.is_signed = b200_type_is_signed_int(cols[c].type);
	t.col = ft_add_col(&A->tc, cols[c].data, t.width);
	if (t.col < 0) {
		return false;
	}
	t.op = op;
	t.value = nodes[r].value.i;
	A->nterms++;
	return true;
}

// the range form of a term whose constant is representable in its column's type (see range_bits)
static void term_range(FilterTerm &t) {
	const int bits = t.width * 8;
	const uint64_t wmask = bits >= 64 ? ~0ULL : ((1ULL << bits) - 1);
	// bit patterns of the type's smallest / largest value
	const uint64_t tmin = t.is_signed ? (1ULL << (bits - 1)) & wmask : 0;
	const uint64_t tmax = t.is_signed ? ((1ULL << (bits - 1)) - 1) : wmask;
	const uint64_t c = (uint64_t)t.value & wmask;
	uint64_t lo = c, hi = c;
	t.neg = 0;
	bool empty = false;
	switch (t.op) {
	case B200_EXPR_EQ:
		break;
	case B200_EXPR_NE:
		t.neg = 1;
		break;
	case B200_EXPR_LT:
		empty = c == tmin;
		lo = tmin;
		hi = (c - 1) & wmask;
		break;
	case B200_EXPR_LE:
		lo = tmin;
		break;
	case B200_EXPR_GT:
		empty = c == tmax;
		lo = (c + 1) & wmask;
		hi = tmax;
		break;
	default: // GE
		hi = tmax;
		break;
	}
	if (empty) { // no value qualifies: the complement of the full range
		lo = tmin;
		hi = tmax;
		t.neg = 1;
	}
	t.lo = lo;
	t.span = (hi - lo) & wmask;
}

// can every term be compared in its column's own type?  (the constant must be representable there)
static int terms_lean(FilterTerm *t, int n) {
	for (int i = 0; i < n; i++) {
		term_range(t[i]);
	}
	for (int i = 0; i < n; i++) {
		int64_t v = t[i].value;
		if (t[i].width >= 8) {
			continue;
		}
		int bits = t[i].width * 8;
		if (t[i].is_signed) {
			if (v < -(1LL << (bits - 1)) || v >= (1LL << (bits - 1))) {
				return 0;
			}
		} else if (v < 0 || v >= (1LL << bits)) {
			return 0;
		}
	}
	return 1;
}

// A': returns B200_OK (launched), B200_ERR_INVALID (not eligible) or a CUDA error
int b200_filter_mask_tile(b200_ctx *ctx, const b200_expr_node *nodes, int filter_root, const DCol *cols, int ncols,
                          uint64_t n, uint32_t *mask32, uint32_t *tile_counts) {
	MaskArgs A;
	memset(&A, 0, sizeof(A));
	if (n == 0 || !collect_terms(nodes, filter_root, cols, ncols, &A) || A.nterms == 0) {
		return B200_ERR_INVALID;
	}
	A.lean = terms_lean(A.t, A.nterms);
	// the largest super-tile (8 K .. 2 K rows) whose three stages fit ~50 KB: four CTAs (32 warps) per SM
	size_t budget = 50 * 1024;
	if (const char *env = getenv("B200_MASK_STAGE_KB")) {
		budget = (size_t)atoi(env) * 1024;
	}
	int mrows = 32;
	for (; mrows > FT_ROWS; mrows >>= 1) {
		tile_cols_finish(&A.tc, (uint32_t)mrows * FT_THREADS);
		if ((size_t)FT_STAGES * A.tc.stage_bytes <= budget) {
			break;
		}
	}
	tile_cols_finish(&A.tc, (uint32_t)mrows * FT_THREADS);
	A.stages = FT_STAGES;
	A.n = n;
	A.mask32 = mask32;
	A.tile_counts = tile_counts;
	size_t smem = (size_t)A.stages * A.tc.stage_bytes;
	if (smem > 200 * 1024) {
		return B200_ERR_INVALID;
	}
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(filter_mask_tile_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(filter_mask_tile_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		CUDA_TRY(cudaFuncSetAttribute(filter_mask_tile_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		attr_set = true;
	}
	uint64_t tile_rows = (uint64_t)mrows * FT_THREADS;
	uint64_t ntiles = (n + tile_rows - 1) / tile_rows;
	int per_sm = (int)((200 * 1024) / (smem + 2048));
	per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
	uint64_t max_grid = (uint64_t)ctx->sm_count * per_sm;
	uint64_t grid = ntiles < max_grid ? ntiles : max_grid;
	switch (mrows) {
	case 32:
		filter_mask_tile_kernel<32><<<(unsigned)grid, FT_THREADS, smem, ctx->stream>>>(A);
		break;
	case 16:
		filter_mask_tile_kernel<16><<<(unsigned)grid, FT_THREADS, smem, ctx->stream>>>(A);
		break;
	default:
		filter_mask_tile_kernel<FT_ROWS><<<(unsigned)grid, FT_THREADS, smem, ctx->stream>>>(A);
		break;
	}
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// C': projections must be plain references to flat non-NULL columns
int b200_filter_compact_tile(b200_ctx *ctx, const b200_expr_node *nodes, const int *proj_roots, int nproj,
                             void *const *out_data, const DCol *cols, int ncols, uint64_t n, const uint32_t *mask32,
                             const uint64_t *tile_offsets, uint32_t *out_sel) {
	CompactArgs A;
	memset(&A, 0, sizeof(A));
	if (n == 0 || nproj > FT_MAX_PROJ) {
		return B200_ERR_INVALID;
	}
	for (int j = 0; j < nproj; j++) {
		const b200_expr_node &nd = nodes[proj_roots[j]];
		if (nd.op != B200_EXPR_COLREF || nd.col < 0 || nd.col >= ncols) {
			return B200_ERR_INVALID;
		}
		const DCol &c = cols[nd.col];
		if (c.vtype != B200_FLAT_VECTOR || c.validity || !tile_ptr_ok(c.data)) {
			return B200_ERR_INVALID;
		}
		A.width[j] = b200_type_size(c.type);
		A.col[j] = ft_add_col(&A.tc, c.data, A.width[j]);
		if (A.col[j] < 0) {
			return B200_ERR_INVALID;
		}
		A.out[j] = out_data[j];
	}
	if (A.tc.n == 0) {
		return B200_ERR_INVALID; // only a selection vector is wanted: the generic kernel handles that
	}
	A.nproj = nproj;
	tile_cols_finish(&A.tc, FT_TILE);
	A.stages = FT_STAGES;
	while (A.stages > 2 && (size_t)A.stages * A.tc.stage_bytes > 100 * 1024) {
		A.stages--;
	}
	A.n = n;
	A.mask32 = mask32;
	A.tile_offsets = tile_offsets;
	A.out_sel = out_sel;
	size_t smem = (size_t)A.stages * A.tc.stage_bytes;
	if (smem > 200 * 1024) {
		return B200_ERR_INVALID;
	}
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(compact_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		attr_set = true;
	}
	uint64_t ntiles = (n + FT_TILE - 1) / FT_TILE;
	int per_sm = (int)((200 * 1024) / (smem + 2048));
	per_sm = per_sm < 1 ? 1 : (per_sm > 6 ? 6 : per_sm);
	uint64_t max_grid = (uint64_t)ctx->sm_count * per_sm;
	uint64_t grid = ntiles < max_grid ? ntiles : max_grid;
	compact_tile_kernel<<<(unsigned)grid, FT_THREADS, smem, ctx->stream>>>(A);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}

// Fused single pass.  out_data[j] must have room for n values (the caller trims to *the count read from total_dev).
// Returns B200_OK (launched), B200_ERR_INVALID (not eligible) or a CUDA error.
int b200_filter_fused_tile(b200_ctx *ctx, const b200_expr_node *nodes, int filter_root, const int *proj_roots, int nproj,
                           void *const *out_data, const DCol *cols, int ncols, uint64_t n, uint32_t *mask32,
                           uint32_t *out_sel, uint32_t *status, unsigned long long *total_dev) {
	FusedArgs A;
	memset(&A, 0, sizeof(A));
	MaskArgs M;
	memset(&M, 0, sizeof(M));
	if (n == 0 || nproj > FT_MAX_PROJ || !collect_terms(nodes, filter_root, cols, ncols, &M) || M.nterms == 0) {
		return B200_ERR_INVALID;
	}
	A.tc = M.tc;
	A.nterms = M.nterms;
	A.lean = terms_lean(M.t, M.nterms);
	for (int i = 0; i < M.nterms; i++) {
		A.t[i] = M.t[i];
	}
	uint32_t cb = 0;
	for (int j = 0; j < nproj; j++) {
		const b200_expr_node &nd = nodes[proj_roots[j]];
		if (nd.op != B200_EXPR_COLREF || nd.col < 0 || nd.col >= ncols) {
			return B200_ERR_INVALID;
		}
		const DCol &c = cols[nd.col];
		if (c.vtype != B200_FLAT_VECTOR || c.validity || !tile_ptr_ok(c.data)) {
			return B200_ERR_INVALID;
		}
		A.width[j] = b200_type_size(c.type);
		A.col[j] = ft_add_col(&A.tc, c.data, A.width[j]);
		if (A.col[j] < 0) {
			return B200_ERR_INVALID;
		}
		A.out[j] = out_data[j];
		A.cbuf_off[j] = cb;
		cb += (uint32_t)A.width[j] * FT_TILE;
	}
	A.nproj = nproj;
	A.sel_off = cb;
	if (out_sel) {
		cb += 4 * FT_TILE;
	}
	tile_cols_finish(&A.tc, FT_TILE);
	// the pipelined kernel needs >= 3 stages (the tile being evaluated, the one being compacted, one in flight)
	A.stages = 4;
	if ((size_t)A.stages * A.tc.stage_bytes + cb > 110 * 1024) {
		A.stages = 3;
	}
	size_t smem = (size_t)A.stages * A.tc.stage_bytes + cb;
	if (smem > 200 * 1024) {
		return B200_ERR_INVALID;
	}
	A.n = n;
	A.mask32 = mask32;
	A.out_sel = out_sel;
	A.status = status;
	A.total = total_dev;
	static bool attr_set = false;
	if (!attr_set) {
		CUDA_TRY(cudaFuncSetAttribute(filter_fused_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
		attr_set = true;
	}
	// the look-back needs every CTA of the grid to be resident: ask the occupancy calculator
	int per_sm = 0;
	CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, filter_fused_tile_kernel, FT_THREADS, smem));
	if (per_sm < 1) {
		return B200_ERR_INVALID;
	}
	per_sm = per_sm > 6 ? 6 : per_sm;
	uint64_t ntiles = (n + FT_TILE - 1) / FT_TILE;
	uint64_t max_grid = (uint64_t)ctx->sm_count * per_sm;
	uint64_t grid = ntiles < max_grid ? ntiles : max_grid;
	filter_fused_tile_kernel<<<(unsigned)grid, FT_THREADS, smem, ctx->stream>>>(A);
	ctx->launches++;
	CUDA_TRY(cudaGetLastError());
	return B200_OK;
}
