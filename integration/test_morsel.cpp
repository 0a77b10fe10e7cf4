// CPU unit test of the binding's host-side staging (B200Staging in b200_binding.hpp): DataChunk columns of every
// vector kind the operators receive - flat, constant, dictionary (sliced), with and without NULLs - must arrive in a
// staging buffer as consecutive values + DuckDB-layout validity words, which is what b200_batch_upload_to ships to
// the GPU.  The buffer is plain host memory laid out by B200Staging::Layout, so no device is needed.
// Built and run by tests/test_integration.py::test_morsel_staging.
#include "b200_binding.hpp"

#include "duckdb/common/types/value.hpp"
#include "duckdb/common/vector/constant_vector.hpp"
#include "duckdb/common/vector/flat_vector.hpp"

#include <cstdio>

using namespace duckdb;

static int failures = 0;
#define CHECK(cond)                                                                                                    \
	do {                                                                                                               \
		if (!(cond)) {                                                                                                 \
			fprintf(stderr, "CHECK failed at line %d: %s\n", __LINE__, #cond);                                         \
			failures++;                                                                                                \
		}                                                                                                              \
	} while (0)

//! a staging ring whose active buffer is host memory, for the columns `infos`
struct HostStaging {
	B200Staging staging;
	vector<uint64_t> memory;
	HostStaging(const vector<B200Column> &infos, idx_t capacity) {
		staging.Layout(infos, capacity);
		memory.assign(staging.bytes / 8 + 1, 0xdeadbeefdeadbeefULL); // garbage where no value was written
		staging.buf[0].base = reinterpret_cast<data_ptr_t>(memory.data());
	}
	template <class T>
	T At(idx_t c, idx_t row) const {
		return reinterpret_cast<const T *>(staging.buf[0].base + staging.data_off[c])[row];
	}
	bool HasValidity(idx_t c) const {
		return staging.buf[0].has_null[c];
	}
	bool Valid(idx_t c, idx_t row) const {
		auto words = reinterpret_cast<const uint64_t *>(staging.buf[0].base + staging.valid_off[c]);
		return !HasValidity(c) || ((words[row >> 6] >> (row & 63)) & 1);
	}
};

//! a DataChunk whose columns reference `vectors`
static void Reference(DataChunk &chunk, vector<Vector *> vectors, idx_t count) {
	vector<LogicalType> types;
	for (auto v : vectors) {
		types.push_back(v->GetType());
	}
	chunk.InitializeEmpty(types);
	for (idx_t c = 0; c < vectors.size(); c++) {
		chunk.data[c].Reference(*vectors[c]);
	}
	chunk.SetCardinalityUnsafe(count);
}

int main() {
	const idx_t n = 100;
	// 1. flat INTEGER with NULLs at i % 7 == 3
	Vector flat(LogicalType::INTEGER, n);
	for (idx_t i = 0; i < n; i++) {
		FlatVector::GetDataMutable<int32_t>(flat)[i] = NumericCast<int32_t>(i * 3) - 50;
		if (i % 7 == 3) {
			FlatVector::SetNull(flat, i, true);
		}
	}
	// 2. flat BIGINT without NULLs
	Vector big(LogicalType::BIGINT, n);
	for (idx_t i = 0; i < n; i++) {
		FlatVector::GetDataMutable<int64_t>(big)[i] = int64_t(i) * 1000000007LL;
	}
	// 3. constant DOUBLE, 4. constant NULL
	Vector constant(Value::DOUBLE(2.5), count_t(n));
	Vector constant_null(Value(LogicalType::SMALLINT), count_t(n));
	// 5. dictionary: a reversed slice of the flat vector (selection i -> n - 1 - i)
	SelectionVector reverse(n);
	for (idx_t i = 0; i < n; i++) {
		reverse.set_index(i, n - 1 - i);
	}
	Vector dict(LogicalType::INTEGER, n);
	dict.Slice(flat, reverse, n);

	{
		HostStaging h({{0, B200_INT32, 4}, {1, B200_INT64, 8}, {2, B200_DOUBLE, 8}, {3, B200_INT16, 2}, {4, B200_INT32, 4}},
		              1024);
		DataChunk chunk;
		Reference(chunk, {&flat, &big, &constant, &constant_null, &dict}, n);
		// two appends (two DataChunks) to cover the offsets of the second one
		h.staging.Append(chunk, 0, n);
		h.staging.Append(chunk, 0, n);
		CHECK(h.staging.buf[0].rows == 2 * n && h.staging.Room() == 1024 - 2 * n);
		for (idx_t row = 0; row < 2 * n; row++) {
			idx_t i = row % n;
			// flat
			CHECK(h.Valid(0, row) == (i % 7 != 3));
			if (i % 7 != 3) {
				CHECK(h.At<int32_t>(0, row) == NumericCast<int32_t>(i * 3) - 50);
			}
			// bigint: no NULLs -> no validity words at all
			CHECK(h.At<int64_t>(1, row) == int64_t(i) * 1000000007LL);
			// constants
			CHECK(h.At<double>(2, row) == 2.5);
			CHECK(!h.Valid(3, row));
			// dictionary = reversed flat
			idx_t src = n - 1 - i;
			CHECK(h.Valid(4, row) == (src % 7 != 3));
			if (src % 7 != 3) {
				CHECK(h.At<int32_t>(4, row) == NumericCast<int32_t>(src * 3) - 50);
			}
		}
		CHECK(!h.HasValidity(1) && !h.HasValidity(2));
		CHECK(h.HasValidity(0) && h.HasValidity(3) && h.HasValidity(4));
	}

	{
		// a column without NULLs in the first append and with NULLs in the second: no validity words until the first
		// NULL, even for a vector with a validity mask, then the rows staged before it must read as valid
		HostStaging h({{0, B200_INT32, 4}}, 1024);
		Vector clean(LogicalType::INTEGER, n);
		for (idx_t i = 0; i < n; i++) {
			FlatVector::GetDataMutable<int32_t>(clean)[i] = NumericCast<int32_t>(i);
		}
		FlatVector::SetNull(clean, 0, true); // a mask whose rows are all valid
		FlatVector::SetNull(clean, 0, false);
		DataChunk first, second;
		Reference(first, {&clean}, n);
		Reference(second, {&flat}, n);
		h.staging.Append(first, 0, n);
		CHECK(!h.HasValidity(0));
		h.staging.Append(second, 0, n);
		CHECK(h.HasValidity(0));
		for (idx_t row = 0; row < 2 * n; row++) {
			bool nulls = row >= n && (row - n) % 7 == 3;
			CHECK(h.Valid(0, row) == !nulls);
			if (!nulls) {
				CHECK(h.At<int32_t>(0, row) ==
				      (row < n ? NumericCast<int32_t>(row) : NumericCast<int32_t>((row - n) * 3) - 50));
			}
		}
	}

	{
		// appends of rows [from, from + count) with from > 0, the second crossing the 64-row validity word
		HostStaging h({{0, B200_INT32, 4}, {4, B200_INT32, 4}}, 1024);
		DataChunk chunk;
		Reference(chunk, {&flat, &big, &constant, &constant_null, &dict}, n);
		h.staging.Append(chunk, 5, 30);  // staged rows 0..29 = rows 5..34
		h.staging.Append(chunk, 40, 60); // staged rows 30..89 = rows 40..99
		CHECK(h.staging.buf[0].rows == 90);
		for (idx_t row = 0; row < 90; row++) {
			idx_t i = row < 30 ? row + 5 : row + 10;
			CHECK(h.Valid(0, row) == (i % 7 != 3));
			if (i % 7 != 3) {
				CHECK(h.At<int32_t>(0, row) == NumericCast<int32_t>(i * 3) - 50);
			}
			idx_t src = n - 1 - i;
			CHECK(h.Valid(1, row) == (src % 7 != 3));
			if (src % 7 != 3) {
				CHECK(h.At<int32_t>(1, row) == NumericCast<int32_t>(src * 3) - 50);
			}
		}
	}

	// eligibility analysis helpers used by the decorators: PhysicalType -> b200_type
	int32_t type = 0;
	CHECK(B200Type(PhysicalType::INT64, type) && type == B200_INT64);
	CHECK(B200Type(PhysicalType::DOUBLE, type) && type == B200_DOUBLE);
	CHECK(!B200Type(PhysicalType::VARCHAR, type) && !B200Type(PhysicalType::INT128, type));

	if (failures) {
		fprintf(stderr, "%d checks failed\n", failures);
		return 1;
	}
	printf("morsel staging OK\n");
	return 0;
}
