// What the operators of the DuckDB-side binding share (see INTEGRATION.md): timing, the status-code and type
// mappings, the pinned staging ring that carries DataChunk columns to the device, the pools behind it, the state of
// an operator that buffers its input into batches, and the decorators' source / local sink states.
// b200_filter.cpp, b200_aggregate.cpp and b200_join.cpp each include this header and compile on their own;
// b200_extension.cpp includes the three into one translation unit.
#pragma once

#include "duckdb/common/exception.hpp"
#include "duckdb/common/types/data_chunk.hpp"
#include "duckdb/common/vector/unified_vector_format.hpp"
#include "duckdb/execution/physical_operator_states.hpp"
#include "duckdb/main/client_context.hpp"

#include "duckdb_b200.h"

#include <cuda_runtime_api.h>

#include <atomic>
#include <chrono>
#include <mutex>

namespace duckdb {

//! B200_TIMING=1: wall-clock nanoseconds per phase of the binding, summed over all worker threads and printed (and
//! reset) by B200TimingReport() when an operator's global state is destroyed - where the time of a query goes between
//! DuckDB's chunks and the kernels.
enum B200Phase : int {
	B200_T_CTX = 0, B200_T_STAGING_INIT, B200_T_APPEND, B200_T_COPY_CHUNK, B200_T_UPLOAD, B200_T_UPLOAD_WAIT, B200_T_LOCK_WAIT,
	B200_T_KERNEL_CALL, B200_T_DOWNLOAD, B200_T_FINALIZE, B200_T_EMIT, B200_T_PHASES
};
static std::atomic<uint64_t> g_b200_ns[B200_T_PHASES];
static std::atomic<uint64_t> g_b200_calls[B200_T_PHASES];
static bool B200TimingOn() {
	static const bool on = getenv("B200_TIMING") != nullptr;
	return on;
}
struct B200Timer {
	int phase;
	std::chrono::steady_clock::time_point t0;
	explicit B200Timer(int phase_p) : phase(phase_p) {
		if (B200TimingOn()) {
			t0 = std::chrono::steady_clock::now();
		}
	}
	~B200Timer() {
		if (B200TimingOn()) {
			auto ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
			g_b200_ns[phase] += uint64_t(ns);
			g_b200_calls[phase]++;
		}
	}
};
static void B200TimingReport(const char *what) {
	if (!B200TimingOn()) {
		return;
	}
	static const char *names[B200_T_PHASES] = {"ctx_create", "staging_init", "append", "copy_chunk", "upload_submit",
	                                           "upload_wait", "lock_wait", "kernel_call", "download", "finalize", "emit"};
	fprintf(stderr, "[b200 timing] %s:", what);
	for (int i = 0; i < B200_T_PHASES; i++) {
		uint64_t ns = g_b200_ns[i].exchange(0), calls = g_b200_calls[i].exchange(0);
		if (calls) {
			fprintf(stderr, " %s=%.2fms/%llu", names[i], double(ns) / 1e6, (unsigned long long)calls);
		}
	}
	fprintf(stderr, "\n");
}

static void B200Check(int rc) {
	if (rc == B200_OK) {
		return;
	}
	// SURVEY.md 8b "Error convention": status codes become duckdb::Exception subclasses
	if (rc == B200_ERR_OVERFLOW) {
		throw OutOfRangeException(string(b200_last_error()));
	}
	if (rc == B200_ERR_OOM) {
		throw OutOfMemoryException(string(b200_last_error()));
	}
	throw IOException("b200: " + string(b200_last_error()));
}

//! PhysicalType -> b200_type (identical numeric values by construction, include/duckdb_b200.h)
static bool B200Type(PhysicalType t, int32_t &out) {
	switch (t) {
	case PhysicalType::BOOL:
	case PhysicalType::UINT8:
	case PhysicalType::INT8:
	case PhysicalType::UINT16:
	case PhysicalType::INT16:
	case PhysicalType::UINT32:
	case PhysicalType::INT32:
	case PhysicalType::UINT64:
	case PhysicalType::INT64:
	case PhysicalType::FLOAT:
	case PhysicalType::DOUBLE:
		out = static_cast<int32_t>(t);
		return true;
	default:
		return false; // VARCHAR, HUGEINT, nested: stock operator
	}
}

struct B200Column {
	idx_t chunk_col;       // column of the input DataChunk
	int32_t type;          // b200_type
	idx_t width;           // bytes
};

static constexpr idx_t B200_MORSEL_ROWS = 1 << 20;

//! What one worker needs to stream morsels to the device: a context (= a CUDA stream), two pinned host buffers and two
//! device buffers of the same size.  Creating these is expensive (stream + page-locking + cudaMalloc: ~5-10 ms per
//! worker, 16 workers per operator, every query) and they are perfectly reusable, so released sets go to a process-wide
//! pool and the next operator state picks one up - per query the row path then contains no allocation at all.
struct B200StagingResources {
	b200_ctx *ctx = nullptr;
	data_ptr_t host[2] = {nullptr, nullptr};
	data_ptr_t dev[2] = {nullptr, nullptr};
	idx_t bytes = 0;

	~B200StagingResources() {
		for (int i = 0; i < 2; i++) {
			if (dev[i]) {
				cudaFree(dev[i]);
			}
			if (host[i]) {
				b200_host_free(ctx, host[i]);
			}
		}
		if (ctx) {
			b200_ctx_destroy(ctx);
		}
	}
};

class B200StagingPool {
public:
	static unique_ptr<B200StagingResources> Acquire(int device, idx_t bytes) {
		{
			std::lock_guard<std::mutex> guard(Lock());
			auto &pool = Pool();
			idx_t best = pool.size();
			for (idx_t i = 0; i < pool.size(); i++) {
				if (pool[i]->bytes >= bytes && pool[i]->bytes <= 4 * bytes + (idx_t(1) << 20) &&
				    (best == pool.size() || pool[i]->bytes < pool[best]->bytes)) {
					best = i;
				}
			}
			if (best != pool.size()) {
				auto res = std::move(pool[best]);
				pool.erase(pool.begin() + NumericCast<int64_t>(best));
				return res;
			}
		}
		auto res = make_uniq<B200StagingResources>();
		{
			B200Timer timer(B200_T_CTX);
			B200Check(b200_ctx_create(device, nullptr, &res->ctx));
		}
		B200Timer timer(B200_T_STAGING_INIT);
		res->bytes = bytes;
		for (int i = 0; i < 2; i++) {
			void *p = nullptr;
			B200Check(b200_host_alloc(res->ctx, bytes, &p));
			res->host[i] = data_ptr_cast(p);
			void *d = nullptr;
			if (cudaMalloc(&d, bytes) != cudaSuccess) {
				throw OutOfMemoryException("b200: cannot allocate the device side of the morsel ring");
			}
			res->dev[i] = data_ptr_cast(d);
		}
		return res;
	}
	static void Release(unique_ptr<B200StagingResources> res) {
		if (!res) {
			return;
		}
		b200_ctx_sync(res->ctx); // nothing of the finished query is still in flight on this stream
		std::lock_guard<std::mutex> guard(Lock());
		if (Pool().size() < 96) {
			Pool().push_back(std::move(res));
		}
	}

private:
	static std::mutex &Lock() {
		static std::mutex lock;
		return lock;
	}
	static vector<unique_ptr<B200StagingResources>> &Pool() {
		static vector<unique_ptr<B200StagingResources>> pool;
		return pool;
	}
};

//! Contexts of the operators' global states (the aggregate / join object lives on it), pooled for the same reason
class B200ContextPool {
public:
	static b200_ctx *Acquire(int device) {
		{
			std::lock_guard<std::mutex> guard(Lock());
			if (!Pool().empty()) {
				auto ctx = Pool().back();
				Pool().pop_back();
				return ctx;
			}
		}
		B200Timer timer(B200_T_CTX);
		b200_ctx *ctx = nullptr;
		B200Check(b200_ctx_create(device, nullptr, &ctx));
		return ctx;
	}
	static void Release(b200_ctx *ctx) {
		if (!ctx) {
			return;
		}
		b200_ctx_sync(ctx);
		std::lock_guard<std::mutex> guard(Lock());
		if (Pool().size() < 32) {
			Pool().push_back(ctx);
		} else {
			b200_ctx_destroy(ctx);
		}
	}

private:
	static std::mutex &Lock() {
		static std::mutex lock;
		return lock;
	}
	static vector<b200_ctx *> &Pool() {
		static vector<b200_ctx *> pool;
		return pool;
	}
};

//! Pinned, double-buffered staging of one worker thread's morsels (north_star: "DataChunk columns pinned and streamed to
//! HBM in morsel-sized batches").  Chunks are appended column-wise into the ACTIVE pinned buffer; a full buffer is
//! copied asynchronously into ITS device buffer on the worker's own context (= its own CUDA stream) while the following
//! chunks fill the other pinned buffer; the operator consumes an uploaded batch one morsel later.  Workers therefore
//! overlap their H2D copies with each other and with the kernels - the only serialised part is the (short, asynchronous)
//! kernel launch itself.  Host and device rings are persistent (B200StagingPool): nothing is allocated per morsel.
struct B200Staging {
	struct Buffer {
		data_ptr_t base = nullptr;     // pinned host buffer
		data_ptr_t dev_base = nullptr; // its device twin
		idx_t rows = 0;
		vector<bool> has_null;
		b200_batch *batch = nullptr; // upload in flight / done, not yet consumed
	};
	unique_ptr<B200StagingResources> res;
	b200_ctx *ctx = nullptr;
	Buffer buf[2];
	int active = 0;
	idx_t capacity = 0;
	vector<B200Column> infos;
	vector<idx_t> data_off, valid_off; // byte offsets inside a buffer
	idx_t bytes = 0;

	~B200Staging() {
		for (auto &b : buf) {
			if (b.batch) {
				b200_batch_free(b.batch);
			}
		}
		B200StagingPool::Release(std::move(res));
	}

	//! the layout of one buffer (every column's values, then every column's validity words, each 256-byte aligned),
	//! without any device resource
	void Layout(const vector<B200Column> &infos_p, idx_t capacity_rows) {
		infos = infos_p;
		capacity = capacity_rows;
		idx_t off = 0;
		for (auto &c : infos) {
			data_off.push_back(off);
			off += (capacity * c.width + 255) & ~idx_t(255);
		}
		for (idx_t c = 0; c < infos.size(); c++) {
			valid_off.push_back(off);
			off += (((capacity + 63) / 64) * 8 + 255) & ~idx_t(255);
		}
		bytes = off;
		for (int i = 0; i < 2; i++) {
			buf[i].has_null.assign(infos.size(), false);
		}
	}

	void Init(int device, const vector<B200Column> &infos_p, idx_t capacity_rows) {
		Layout(infos_p, capacity_rows);
		res = B200StagingPool::Acquire(device, bytes);
		ctx = res->ctx;
		for (int i = 0; i < 2; i++) {
			buf[i].base = res->host[i];
			buf[i].dev_base = res->dev[i];
		}
	}

	idx_t Room() const {
		return capacity - buf[active].rows;
	}

	//! append rows [from, from + count) of the chunk's columns `chunk_cols` (one per staged column)
	void Append(DataChunk &chunk, idx_t from, idx_t count) {
		B200Timer timer(B200_T_APPEND);
		auto &b = buf[active];
		for (idx_t c = 0; c < infos.size(); c++) {
			auto &vec = chunk.data[infos[c].chunk_col];
			idx_t width = infos[c].width;
			UnifiedVectorFormat format;
			vec.ToUnifiedFormat(format);
			auto dst = b.base + data_off[c] + b.rows * width;
			if (!format.sel->IsSet()) {
				memcpy(dst, format.data + from * width, count * width); // flat vector: rows are already consecutive
			} else {
				for (idx_t i = 0; i < count; i++) {
					memcpy(dst + i * width, format.data + format.sel->get_index(from + i) * width, width);
				}
			}
			// validity words only once the morsel holds a NULL: an all-valid mask would cost the kernels their NULL-free
			// paths (the dense join table, for one, only inlines payloads without a mask)
			bool nullable = format.validity.CanHaveNull();
			auto words = reinterpret_cast<uint64_t *>(b.base + valid_off[c]);
			for (idx_t i = 0; i < count && nullable && !b.has_null[c]; i++) {
				if (!format.validity.RowIsValid(format.sel->get_index(from + i))) {
					// first NULL of this morsel: every row so far is valid
					for (idx_t w = 0; w < (b.rows + 63) / 64; w++) {
						words[w] = ~uint64_t(0);
					}
					b.has_null[c] = true;
				}
			}
			if (b.has_null[c]) {
				for (idx_t i = 0; i < count; i++) {
					idx_t row = b.rows + i;
					bool valid = !nullable || format.validity.RowIsValid(format.sel->get_index(from + i));
					uint64_t bit = uint64_t(1) << (row & 63);
					if ((row & 63) == 0) {
						words[row >> 6] = 0;
					}
					words[row >> 6] = valid ? (words[row >> 6] | bit) : (words[row >> 6] & ~bit);
				}
			}
		}
		b.rows += count;
	}

	//! the batch uploaded one morsel ago (its copy has completed), or nullptr
	b200_batch *TakeUploaded() {
		auto &other = buf[1 - active];
		if (!other.batch) {
			return nullptr;
		}
		{
			B200Timer timer(B200_T_UPLOAD_WAIT);
			B200Check(b200_ctx_sync(ctx)); // only that upload is on this stream
		}
		auto batch = other.batch;
		other.batch = nullptr;
		other.rows = 0;
		other.has_null.assign(infos.size(), false);
		return batch;
	}

	//! start the asynchronous upload of the active buffer and switch buffers (the other one must have been taken)
	void SubmitActive() {
		auto &b = buf[active];
		if (b.rows == 0) {
			return;
		}
		vector<b200_vector> cols(infos.size());
		vector<void *> dev_data(infos.size()), dev_valid(infos.size());
		for (idx_t c = 0; c < infos.size(); c++) {
			cols[c].type = infos[c].type;
			cols[c].vector_type = B200_FLAT_VECTOR;
			cols[c].data = b.base + data_off[c];
			cols[c].sel = nullptr;
			cols[c].validity = b.has_null[c] ? reinterpret_cast<uint64_t *>(b.base + valid_off[c]) : nullptr;
			cols[c].dict_size = 0;
			dev_data[c] = b.dev_base + data_off[c];
			dev_valid[c] = b.dev_base + valid_off[c];
		}
		{
			B200Timer timer(B200_T_UPLOAD);
			B200Check(b200_batch_upload_to(ctx, cols.data(), NumericCast<int>(cols.size()), b.rows, dev_data.data(),
			                               dev_valid.data(), &b.batch));
		}
		active = 1 - active;
	}

	//! Sink: append the chunk; whenever the active buffer is full, sink(batch) consumes the morsel uploaded while this
	//! one was being filled (nullptr for the first), then the full buffer starts its upload
	template <class SINK>
	void Feed(DataChunk &chunk, SINK &&sink) {
		idx_t from = 0;
		while (from < chunk.size()) {
			idx_t count = MinValue<idx_t>(chunk.size() - from, Room());
			Append(chunk, from, count);
			from += count;
			if (Room() == 0) {
				sink(TakeUploaded());
				SubmitActive();
			}
		}
	}

	//! Combine: sink(batch) the morsel in flight and the partial one
	template <class SINK>
	void Drain(SINK &&sink) {
		sink(TakeUploaded());
		SubmitActive();
		sink(TakeUploaded());
	}
};

//! Operator state of an operator that runs its kernel on batches of buffered input (the join probe, the filter): input
//! chunks are kept as deep copies (their vectors back the output slices) and the columns the kernel reads are staged in
//! the worker's ring until the batch is full; ONE kernel call handles the batch, and its result is emitted chunk by
//! chunk (HAVE_MORE_OUTPUT, then FinalExecute for the last, partial batch).  Kernel calls per chunk would be one
//! synchronous H2D -> kernel -> D2H round trip per 2048 rows.
class B200BatchState : public OperatorState {
public:
	~B200BatchState() override {
		if (sel_dev) {
			cudaFree(sel_dev);
		}
	}
	B200Staging staging;                    // the kernel's columns of the buffered rows (pinned, own stream)
	vector<unique_ptr<DataChunk>> buffered; // copies of the buffered input chunks (their vectors back the output slices)
	vector<idx_t> chunk_start;              // first batch row of every buffered chunk
	idx_t buffered_rows = 0;
	bool input_taken = false;               // the current input chunk is already in the buffer
	bool draining = false;                  // the result of the last batch is being emitted
	idx_t emit_chunk = 0, emit_pos = 0;     // emit cursor: buffered chunk, position in its result
	uint32_t *sel_dev = nullptr;            // device buffer for one batch row id per result row
	idx_t sel_capacity = 0;

	//! keep a copy of the input chunk and stage the kernel's columns
	void Buffer(ClientContext &context, DataChunk &input) {
		if (input.size() == 0) {
			return;
		}
		auto copy = make_uniq<DataChunk>();
		{
			B200Timer timer(B200_T_COPY_CHUNK);
			copy->Initialize(Allocator::Get(context), input.GetTypes());
			input.Copy(*copy);
		}
		staging.Append(*copy, 0, copy->size());
		chunk_start.push_back(buffered_rows);
		buffered_rows += copy->size();
		buffered.push_back(std::move(copy));
	}

	//! room for `rows` row ids in sel_dev; on failure `batch` is freed and OutOfMemoryException is thrown
	void ReserveSel(idx_t rows, b200_batch *batch) {
		if (sel_capacity >= rows) {
			return;
		}
		if (sel_dev) {
			cudaFree(sel_dev);
			sel_dev = nullptr;
		}
		sel_capacity = rows + rows / 4 + 1024;
		if (cudaMalloc(reinterpret_cast<void **>(&sel_dev), sel_capacity * sizeof(uint32_t)) != cudaSuccess) {
			sel_dev = nullptr;
			sel_capacity = 0;
			b200_batch_free(batch);
			throw OutOfMemoryException("b200: cannot allocate the device selection buffer");
		}
	}

	//! release a drained batch
	void Reset() {
		buffered.clear();
		chunk_start.clear();
		buffered_rows = 0;
		draining = false;
	}

	//! PhysicalOperator::Execute: buffer the input; once `batch_rows` rows are buffered, run(batch) makes the kernel
	//! call on the uploaded batch; emit(chunk) then produces the next output chunk, false when the batch is drained
	template <class RUN, class EMIT>
	OperatorResultType Execute(ExecutionContext &context, DataChunk &input, DataChunk &chunk, idx_t batch_rows, RUN &&run,
	                           EMIT &&emit) {
		if (!input_taken) {
			Buffer(context.client, input);
			input_taken = true;
			if (buffered_rows >= batch_rows) {
				RunBatch(context, run);
			}
		}
		if (draining && EmitNext(chunk, emit)) {
			return OperatorResultType::HAVE_MORE_OUTPUT; // called again with the same input (already buffered)
		}
		input_taken = false;
		return OperatorResultType::NEED_MORE_INPUT;
	}

	//! PhysicalOperator::FinalExecute: the last, partial batch
	template <class RUN, class EMIT>
	OperatorFinalizeResultType FinalExecute(ExecutionContext &context, DataChunk &chunk, RUN &&run, EMIT &&emit) {
		if (!draining && buffered_rows > 0) {
			RunBatch(context, run);
		}
		if (draining && EmitNext(chunk, emit)) {
			return OperatorFinalizeResultType::HAVE_MORE_OUTPUT;
		}
		return OperatorFinalizeResultType::FINISHED;
	}

private:
	template <class RUN>
	void RunBatch(ExecutionContext &context, RUN &run) {
		context.client.InterruptCheck();
		draining = true;
		emit_chunk = 0;
		emit_pos = 0;
		staging.SubmitActive();      // H2D of the staged columns on this worker's stream
		run(staging.TakeUploaded()); // ... and wait for it (only this worker blocks)
	}

	template <class EMIT>
	bool EmitNext(DataChunk &chunk, EMIT &emit) {
		if (emit(chunk)) {
			return true;
		}
		Reset();
		chunk.SetCardinality(0);
		return false;
	}
};

//! Local sink state of the decorators: the worker's staging ring on a device, the wrapped operator's state without
class B200LocalSinkState : public LocalSinkState {
public:
	B200Staging staging;
	unique_ptr<LocalSinkState> inner;
};

//! Source states of the decorators: the wrapped operator's states without a device
class B200SourceState : public GlobalSourceState {
public:
	idx_t position = 0; // next result row of the aggregate on a device
	unique_ptr<GlobalSourceState> inner;
	idx_t MaxThreads() override {
		return inner ? inner->MaxThreads() : 1;
	}
};

class B200LocalSourceState : public LocalSourceState {
public:
	unique_ptr<LocalSourceState> inner;
};

} // namespace duckdb
