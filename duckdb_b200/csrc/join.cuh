// Shared definitions of the hash-join kernels (join.cu: build + generic probe, join_tile.cu: TMA-staged probe).
#pragma once
#include "common.cuh"

#define MAX_PAYLOAD 12
#define MAX_LHS 12
#define ROW_NONE 0xffffffffu
#define EMPTY_KEY 0x8000000000000000ULL

struct JoinSlot {
	uint64_t key;
	uint32_t head;
	uint32_t inl;
};

struct PayloadStore {
	void *data[MAX_PAYLOAD];
	uint64_t *validity[MAX_PAYLOAD]; // nullptr when no NULL was ever sunk
	int type[MAX_PAYLOAD];
	int n;
};

struct KeyStore {
	uint64_t *data[MAX_KEYS]; // canonical 64-bit key bits, composite keys only
	int n;
};

struct b200_join {
	b200_ctx *ctx;
	int join_type;
	int nkeys;
	int key_type[MAX_KEYS];
	bool exact; // single key column: key64 is the key itself
	PayloadStore ps;
	KeyStore ks;
	uint64_t *hashes;   // per build row: key64 (exact key or hash); EMPTY_KEY-tagged rows flagged in row_null
	uint8_t *row_skip;  // per build row: 1 = NULL key (never inserted)
	uint64_t rows;
	uint64_t capacity_rows;
	bool any_payload_null[MAX_PAYLOAD];
	// table
	JoinSlot *slots;
	uint64_t table_cap; // power of two; slot [table_cap] is the side slot for key == EMPTY_KEY
	uint32_t *next;
	// dense ("perfect hash") table: unique integer keys in a bounded range are direct-addressed
	uint32_t *dense;     // entry = 0 empty | row + 1 | (inline payload << 8) | 1
	uint64_t dense_min;
	uint64_t dense_range;
	bool finalized;
	bool unique;        // no duplicate keys
	bool inline_payload;
	bool has_null_key;
	uint8_t *matched; // RIGHT / OUTER: per build row, 1 once a probe row matched it (allocated by finalize)
	unsigned long long *counters; // device [0]=dup count, [1]=out cursor, [2]=null keys, [3] total matches
};

#ifdef __CUDACC__
__device__ __forceinline__ uint64_t slot_hash(bool exact, int key_type, uint64_t key64) {
	// exact keys: spread with DuckDB's own hash of the key (hash.hpp:38-54); composite: key64 is already a hash
	return exact ? hash_raw(key_type, key64) : key64;
}

// ------------------------------------------------------------------ probe
struct ProbeOut {
	void *lhs_data[MAX_LHS];
	uint64_t *lhs_valid[MAX_LHS];
	DCol lhs_src[MAX_LHS];
	int nlhs;
	void *pay_data[MAX_PAYLOAD];
	uint64_t *pay_valid[MAX_PAYLOAD];
	uint8_t *mark;        // MARK join: BOOL column
	uint64_t *mark_valid;
	uint32_t *lhs_sel;
};

struct JoinView {
	const uint32_t *dense; // non-NULL: direct-addressed table, see b200_join_finalize
	uint64_t dense_min;
	uint64_t dense_range;
	const JoinSlot *slots;
	uint64_t mask;
	const uint32_t *next;
	bool exact;
	bool unique;
	bool inline_payload;
	int nkeys;
	int key_type[MAX_KEYS];
	KeyStore ks;
	PayloadStore ps;
	bool build_has_null;
	bool build_empty;
	uint8_t *matched; // RIGHT / OUTER joins: the probe sets the flag of every build row it emits; NULL otherwise
};

// first build row matching the probe key of `row`, or ROW_NONE; *inl receives the slot's inline payload
__device__ __forceinline__ uint32_t probe_first(const JoinView &J, const KeyCols &keys, uint64_t row, bool *key_null,
                                                uint64_t ckeys[MAX_KEYS], uint32_t *inl) {
	bool nul = false;
	uint64_t key64;
	if (J.exact) {
		const DCol &c = keys.c[0];
		uint64_t idx = col_index(c, row);
		nul = !col_valid_at(c, idx);
		key64 = canonical_key_bits(c.type, col_load_raw(c, idx));
	} else {
		key64 = hash_row(keys, row, &nul);
#pragma unroll 1
		for (int j = 0; j < J.nkeys; j++) {
			const DCol &c = keys.c[j];
			ckeys[j] = canonical_key_bits(c.type, col_load_raw(c, col_index(c, row)));
		}
	}
	*key_null = nul;
	if (nul || J.build_empty) {
		return ROW_NONE;
	}
	if (J.dense) {
		uint64_t idx = key64 - J.dense_min;
		if (idx >= J.dense_range) {
			return ROW_NONE;
		}
		uint32_t e = __ldg(&J.dense[idx]);
		if (!e) {
			return ROW_NONE;
		}
		*inl = e >> 8;
		return J.inline_payload ? 0u : e - 1;
	}
	uint32_t r;
	if (key64 == EMPTY_KEY) {
		const JoinSlot &s = J.slots[J.mask + 1]; // side slot
		*inl = s.inl;
		r = s.head;
	} else {
		uint64_t slot = slot_hash(J.exact, J.key_type[0], key64) & J.mask;
		while (true) {
			// one 16-byte load: key + head + inline payload
			uint4 v = __ldg((const uint4 *)&J.slots[slot]);
			uint64_t k = ((uint64_t)v.y << 32) | v.x;
			if (k == key64) {
				*inl = v.w;
				r = v.z;
				break;
			}
			if (k == EMPTY_KEY) {
				return ROW_NONE;
			}
			slot = (slot + 1) & J.mask;
		}
	}
	if (!J.exact) {
		// verify the composite key along the chain (the slot only matched on the 64-bit hash)
		while (r != ROW_NONE) {
			bool eq = true;
			for (int j = 0; j < J.nkeys; j++) {
				eq = eq && J.ks.data[j][r] == ckeys[j];
			}
			if (eq) {
				break;
			}
			r = J.next[r];
		}
	}
	return r;
}

__device__ __forceinline__ uint32_t chain_next(const JoinView &J, uint32_t r, const uint64_t ckeys[MAX_KEYS]) {
	r = J.next[r];
	if (!J.exact) {
		while (r != ROW_NONE) {
			bool eq = true;
			for (int j = 0; j < J.nkeys; j++) {
				eq = eq && J.ks.data[j][r] == ckeys[j];
			}
			if (eq) {
				break;
			}
			r = J.next[r];
		}
	}
	return r;
}

__device__ __forceinline__ void emit_row(const JoinView &J, const ProbeOut &po, uint64_t opos, uint64_t prow,
                                         uint32_t brow, uint32_t inl, bool with_payload) {
	if (po.lhs_sel) {
		po.lhs_sel[opos] = (uint32_t)prow;
	}
	for (int j = 0; j < po.nlhs; j++) {
		const DCol &c = po.lhs_src[j];
		uint64_t idx = col_index(c, prow);
		store_raw(po.lhs_data[j], c.type, opos, col_load_raw(c, idx));
		if (po.lhs_valid[j] && !col_valid_at(c, idx)) {
			atomicAnd((unsigned long long *)&po.lhs_valid[j][opos >> 6], ~(1ULL << (opos & 63)));
		}
	}
	if (!with_payload) {
		return;
	}
	if (brow == ROW_NONE) {
		// LEFT join, no partner: NULL payload
		for (int p = 0; p < J.ps.n; p++) {
			store_raw(po.pay_data[p], J.ps.type[p], opos, 0);
			atomicAnd((unsigned long long *)&po.pay_valid[p][opos >> 6], ~(1ULL << (opos & 63)));
		}
		return;
	}
	if (J.inline_payload) {
		int sh = 0;
		for (int p = 0; p < J.ps.n; p++) {
			int sz = b200_type_size(J.ps.type[p]);
			uint32_t bits = inl >> sh;
			sh += sz * 8;
			uint64_t raw = bits;
			if (sz == 1) {
				raw = b200_type_is_signed_int(J.ps.type[p]) ? (uint64_t)(int64_t)(int8_t)bits : (bits & 0xff);
			} else if (sz == 2) {
				raw = b200_type_is_signed_int(J.ps.type[p]) ? (uint64_t)(int64_t)(int16_t)bits : (bits & 0xffff);
			}
			store_raw(po.pay_data[p], J.ps.type[p], opos, raw);
		}
		return;
	}
	for (int p = 0; p < J.ps.n; p++) {
		DCol c;
		c.data = J.ps.data[p];
		c.type = J.ps.type[p];
		c.sel = nullptr;
		c.validity = J.ps.validity[p];
		c.vtype = B200_FLAT_VECTOR;
		store_raw(po.pay_data[p], c.type, opos, col_load_raw(c, brow));
		if (po.pay_valid[p] && !col_valid_at(c, brow)) {
			atomicAnd((unsigned long long *)&po.pay_valid[p][opos >> 6], ~(1ULL << (opos & 63)));
		}
	}
}

#endif
