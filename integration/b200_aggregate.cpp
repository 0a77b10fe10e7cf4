// Reference-side binding of the hash aggregate (see INTEGRATION.md): B200HashAggregate, a sink + source
// PhysicalOperator that DECORATES the stock PhysicalHashAggregate the reference's planner produced.
//
//   replaces PhysicalHashAggregate::{Sink,Combine,Finalize,GetDataInternal}
//            (src/execution/operator/aggregate/physical_hash_aggregate.cpp:415,503,838,958)
//
// The stock operator is planned as usual (so groups / aggregates are already reduced to BOUND_REFs of the child
// chunk, plan_aggregate.cpp:313+); when its shape is eligible - one grouping set, no DISTINCT / FILTER, group and
// aggregate inputs of numeric physical types, aggregates in {count_star, count, sum, sum_no_overflow, min, max,
// avg} - it is wrapped.  With a CUDA device the wrapper batches the 2048-row chunks into morsels, uploads them
// and calls b200_agg_sink; Finalize downloads [groups..., results...] and GetData emits them in <= 2048-row
// chunks.  Without a device ("plumbing, no GPU") every call is forwarded to the wrapped stock operator.
// Ineligible aggregates are not wrapped at all (the plan keeps the stock operator).
#include "duckdb/execution/operator/aggregate/physical_hash_aggregate.hpp"
#include "duckdb/planner/expression/bound_aggregate_expression.hpp"
#include "duckdb/planner/expression/bound_reference_expression.hpp"
#include "duckdb/common/types/hugeint.hpp"
#include "duckdb/common/vector/flat_vector.hpp"
#include "duckdb/common/vector/unified_vector_format.hpp"

#include <mutex>

namespace duckdb {

struct B200Column {
	idx_t chunk_col;       // column of the input DataChunk
	int32_t type;          // b200_type
	idx_t width;           // bytes
};

struct B200AggResult {
	enum Kind { DIRECT, INT128_TO_RESULT, AVG_INT } kind;
	int desc;       // index of the b200 aggregate (AVG_INT: the SUM, desc + 1 is the COUNT)
	double scale;   // AVG over DECIMAL: 10^scale, else 1
	bool int16;     // AVG_INT over an INT16 input (SMALLINT, DECIMAL(<=4)): divided in double, not long double
};

struct B200AggPlan {
	bool eligible = false;
	vector<B200Column> groups;
	vector<B200Column> inputs; // distinct aggregate inputs
	vector<b200_agg_desc> descs;
	vector<B200AggResult> results; // one per DuckDB aggregate
};

static B200AggPlan AnalyseAggregate(const PhysicalHashAggregate &op) {
	B200AggPlan plan;
	auto &data = op.grouped_aggregate_data;
	if (op.grouping_sets.size() != 1 || op.distinct_collection_info || data.groups.empty() ||
	    !data.grouping_functions.empty() || data.groups.size() > 8 || data.aggregates.size() > 12) {
		return plan;
	}
	for (auto &group : data.groups) {
		int32_t type;
		if (group->GetExpressionClass() != ExpressionClass::BOUND_REF ||
		    !B200Type(group->GetReturnType().InternalType(), type)) {
			return plan;
		}
		plan.groups.push_back({group->Cast<BoundReferenceExpression>().Index(), type, GetTypeIdSize(group->GetReturnType().InternalType())});
	}
	for (auto &expr : data.aggregates) {
		auto &aggr = expr->Cast<BoundAggregateExpression>();
		if (aggr.IsDistinct() || aggr.GetFilter() || aggr.GetChildren().size() > 1) {
			return plan;
		}
		auto name = aggr.Function().GetName().GetIdentifierName();
		B200AggResult res {B200AggResult::DIRECT, NumericCast<int>(plan.descs.size()), 1.0, false};
		if (name == "count_star") {
			plan.descs.push_back({B200_AGG_COUNT_STAR, B200_INT64, -1, 0});
			plan.results.push_back(res);
			continue;
		}
		if (aggr.GetChildren().size() != 1 || aggr.GetChildren()[0]->GetExpressionClass() != ExpressionClass::BOUND_REF) {
			return plan;
		}
		auto &child = aggr.GetChildren()[0];
		int32_t in_type;
		if (!B200Type(child->GetReturnType().InternalType(), in_type)) {
			return plan;
		}
		idx_t col = child->Cast<BoundReferenceExpression>().Index();
		int input = -1;
		for (idx_t i = 0; i < plan.inputs.size(); i++) {
			if (plan.inputs[i].chunk_col == col) {
				input = NumericCast<int>(i);
			}
		}
		if (input < 0) {
			input = NumericCast<int>(plan.inputs.size());
			plan.inputs.push_back({col, in_type, GetTypeIdSize(child->GetReturnType().InternalType())});
		}
		bool is_float = in_type == B200_FLOAT || in_type == B200_DOUBLE;
		auto result_physical = expr->GetReturnType().InternalType();
		if (name == "count") {
			plan.descs.push_back({B200_AGG_COUNT, in_type, input, 0});
		} else if (name == "sum" || name == "sum_no_overflow") {
			plan.descs.push_back({B200_AGG_SUM, in_type, input, 0});
			if (is_float) {
				if (in_type != B200_DOUBLE || result_physical != PhysicalType::DOUBLE) {
					return plan;
				}
			} else {
				// SUM(int) comes back as INT128; the reference's result is HUGEINT / DECIMAL(38) or, for the
				// no-overflow variants, BIGINT / DECIMAL(18): keep 128 or the low 64 bits
				if (result_physical != PhysicalType::INT128 && result_physical != PhysicalType::INT64) {
					return plan;
				}
				res.kind = B200AggResult::INT128_TO_RESULT;
			}
		} else if (name == "min" || name == "max") {
			plan.descs.push_back({name == "min" ? B200_AGG_MIN : B200_AGG_MAX, in_type, input, 0});
		} else if (name == "avg") {
			// only the AVGs that return a DOUBLE: over TIMESTAMP / TIME (and their _TZ forms) the result is of the input
			// type, rounded by integer division (DiscreteAverageOperation, avg.cpp:127-144)
			if (result_physical != PhysicalType::DOUBLE) {
				return plan;
			}
			if (is_float) {
				if (in_type != B200_DOUBLE) {
					return plan;
				}
				plan.descs.push_back({B200_AGG_AVG, in_type, input, 0});
			} else {
				// INT16: IntegerAverageOperation::Finalize (avg.cpp:93-107), double(sum) / (double(count) * scale);
				// INT32 / INT64: IntegerAverageOperationHugeint::Finalize (avg.cpp:109-121), the same in long double
				plan.descs.push_back({B200_AGG_SUM, in_type, input, 0});
				plan.descs.push_back({B200_AGG_COUNT, in_type, input, 0});
				res.kind = B200AggResult::AVG_INT;
				res.int16 = in_type == B200_INT16;
				if (child->GetReturnType().id() == LogicalTypeId::DECIMAL) {
					res.scale = std::pow(10.0, double(DecimalType::GetScale(child->GetReturnType())));
				}
			}
		} else {
			return plan;
		}
		plan.results.push_back(res);
	}
	// limits of b200_agg_create (MAX_AGGS / MAX_INPUTS / packed key bytes, csrc/agg.cuh)
	idx_t key_bytes = 0;
	for (auto &g : plan.groups) {
		if ((key_bytes & 7) + g.width > 8) {
			key_bytes = (key_bytes + 7) & ~idx_t(7); // a field never straddles a 64-bit word
		}
		key_bytes += g.width;
	}
	if (plan.descs.size() > 16 || plan.inputs.size() > 12 || key_bytes + 1 > 32) {
		return plan;
	}
	plan.eligible = true;
	return plan;
}

//! a host-side morsel: flattened copies of the needed columns of many DataChunks
struct B200Morsel {
	vector<vector<data_t>> data;
	vector<vector<uint8_t>> valid; // one byte per row (packed into validity words at flush time)
	vector<bool> has_null;
	idx_t rows = 0;

	void Init(idx_t ncols) {
		data.resize(ncols);
		valid.resize(ncols);
		has_null.assign(ncols, false);
	}
	//! flat b200_vector views of the buffered columns (validity words only for columns that saw a NULL)
	void ToVectors(const vector<B200Column> &infos, vector<b200_vector> &cols, vector<vector<uint64_t>> &masks) {
		idx_t ncols = data.size();
		cols.resize(ncols);
		masks.resize(ncols);
		for (idx_t c = 0; c < ncols; c++) {
			cols[c].type = infos[c].type;
			cols[c].vector_type = B200_FLAT_VECTOR;
			cols[c].data = data[c].data();
			cols[c].sel = nullptr;
			cols[c].validity = nullptr;
			cols[c].dict_size = 0;
			if (has_null[c]) {
				masks[c].assign((rows + 63) / 64, 0);
				for (idx_t i = 0; i < rows; i++) {
					if (valid[c][i]) {
						masks[c][i >> 6] |= uint64_t(1) << (i & 63);
					}
				}
				cols[c].validity = masks[c].data();
			}
		}
	}
	void Clear() {
		for (idx_t c = 0; c < data.size(); c++) {
			data[c].clear();
			valid[c].clear();
			has_null[c] = false;
		}
		rows = 0;
	}
	//! append `count` rows of a DataChunk column (flat / constant / dictionary / sliced): values are gathered through
	//! the selection of the unified format, NULL rows keep whatever bytes the vector holds and clear their flag
	void Append(Vector &vec, idx_t col, idx_t count, idx_t width) {
		UnifiedVectorFormat format;
		vec.ToUnifiedFormat(format);
		auto &d = data[col];
		auto &v = valid[col];
		idx_t old = d.size();
		d.resize(old + count * width);
		v.resize(rows + count, 1);
		auto dst = d.data() + old;
		if (!format.sel->IsSet()) {
			memcpy(dst, format.data, count * width); // flat vector: rows are already consecutive
		} else {
			for (idx_t i = 0; i < count; i++) {
				memcpy(dst + i * width, format.data + format.sel->get_index(i) * width, width);
			}
		}
		if (format.validity.CanHaveNull()) {
			for (idx_t i = 0; i < count; i++) {
				if (!format.validity.RowIsValid(format.sel->get_index(i))) {
					v[rows + i] = 0;
					has_null[col] = true;
				}
			}
		}
	}
};


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

	void Init(int device, const vector<B200Column> &infos_p, idx_t capacity_rows) {
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
		res = B200StagingPool::Acquire(device, bytes);
		ctx = res->ctx;
		for (int i = 0; i < 2; i++) {
			buf[i].base = res->host[i];
			buf[i].dev_base = res->dev[i];
			buf[i].has_null.assign(infos.size(), false);
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
			if (format.validity.CanHaveNull()) {
				auto words = reinterpret_cast<uint64_t *>(b.base + valid_off[c]);
				if (!b.has_null[c]) {
					// first NULL-able vector of this morsel: every row so far is valid
					for (idx_t w = 0; w < (b.rows + 63) / 64; w++) {
						words[w] = ~uint64_t(0);
					}
					b.has_null[c] = true;
				}
				for (idx_t i = 0; i < count; i++) {
					idx_t row = b.rows + i;
					bool valid = format.validity.RowIsValid(format.sel->get_index(from + i));
					uint64_t bit = uint64_t(1) << (row & 63);
					if ((row & 63) == 0) {
						words[row >> 6] = 0;
					}
					words[row >> 6] = valid ? (words[row >> 6] | bit) : (words[row >> 6] & ~bit);
				}
			} else if (b.has_null[c]) {
				auto words = reinterpret_cast<uint64_t *>(b.base + valid_off[c]);
				for (idx_t i = 0; i < count; i++) {
					idx_t row = b.rows + i;
					if ((row & 63) == 0) {
						words[row >> 6] = 0;
					}
					words[row >> 6] |= uint64_t(1) << (row & 63);
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
};

class B200AggGlobalState : public GlobalSinkState {
public:
	std::mutex lock;
	b200_ctx *ctx = nullptr;
	b200_agg *agg = nullptr;
	// results on the host: [groups..., b200 aggregates...]
	vector<vector<data_t>> result_data;
	vector<vector<uint64_t>> result_valid;
	idx_t result_rows = 0;
	bool finalized = false;

	~B200AggGlobalState() override {
		B200TimingReport("hash aggregate");
		if (agg) {
			b200_agg_destroy(agg);
		}
		B200ContextPool::Release(ctx);
	}
};

class B200AggLocalState : public LocalSinkState {
public:
	B200Staging staging;
	unique_ptr<LocalSinkState> inner;
};

class B200AggSourceState : public GlobalSourceState {
public:
	idx_t position = 0;
	unique_ptr<GlobalSourceState> inner;
	idx_t MaxThreads() override {
		return inner ? inner->MaxThreads() : 1;
	}
};

class B200AggLocalSourceState : public LocalSourceState {
public:
	unique_ptr<LocalSourceState> inner;
};

static constexpr idx_t B200_MORSEL_ROWS = 1 << 20;

class B200HashAggregate : public PhysicalOperator {
public:
	B200HashAggregate(PhysicalPlan &physical_plan, PhysicalHashAggregate &inner_p, B200AggPlan plan_p)
	    : PhysicalOperator(physical_plan, PhysicalOperatorType::EXTENSION, inner_p.types, inner_p.estimated_cardinality),
	      inner(inner_p), plan(std::move(plan_p)), on_device(b200_device_count() > 0) {
		for (auto &child : inner_p.children) {
			children.push_back(child);
		}
	}

	PhysicalHashAggregate &inner; // the stock operator this one decorates (lives in the same plan arena)
	B200AggPlan plan;
	bool on_device;

	string GetName() const override {
		return on_device ? "B200_HASH_GROUP_BY" : "B200_HASH_GROUP_BY(host)";
	}
	InsertionOrderPreservingMap<string> ParamsToString() const override {
		auto result = inner.ParamsToString();
		result["Operator"] = GetName();
		return result;
	}

	// ------------------------------------------------------------------ sink
	bool IsSink() const override {
		return true;
	}
	bool ParallelSink() const override {
		return true;
	}
	bool SinkOrderDependent() const override {
		return false;
	}

	unique_ptr<GlobalSinkState> GetGlobalSinkState(ClientContext &context) const override {
		auto state = make_uniq<B200AggGlobalState>();
		if (!on_device) {
			inner.sink_state = inner.GetGlobalSinkState(context);
			return std::move(state);
		}
		state->ctx = B200ContextPool::Acquire(0);
		vector<int32_t> key_types;
		for (auto &g : plan.groups) {
			key_types.push_back(g.type);
		}
		B200Check(b200_agg_create(state->ctx, key_types.data(), NumericCast<int>(key_types.size()), plan.descs.data(),
		                          NumericCast<int>(plan.descs.size()), 0, &state->agg));
		return std::move(state);
	}

	unique_ptr<LocalSinkState> GetLocalSinkState(ExecutionContext &context) const override {
		auto state = make_uniq<B200AggLocalState>();
		if (!on_device) {
			state->inner = inner.GetLocalSinkState(context);
		} else {
			vector<B200Column> infos = plan.groups;
			infos.insert(infos.end(), plan.inputs.begin(), plan.inputs.end());
			state->staging.Init(0, infos, B200_MORSEL_ROWS);
		}
		return std::move(state);
	}

	//! sink one uploaded batch: the aggregate object lives on the global context and is driven by one thread at a time
	void SinkBatch(ExecutionContext &context, B200AggGlobalState &g, b200_batch *batch) const {
		if (!batch) {
			return;
		}
		context.client.InterruptCheck(); // long-running sinks stay cancellable (aggregate_hashtable.cpp:1183)
		vector<int> key_cols, input_cols;
		idx_t ncols = plan.groups.size() + plan.inputs.size();
		for (idx_t c = 0; c < ncols; c++) {
			(c < plan.groups.size() ? key_cols : input_cols).push_back(NumericCast<int>(c));
		}
		int rc;
		{
			auto t_lock = make_uniq<B200Timer>(B200_T_LOCK_WAIT);
			std::lock_guard<std::mutex> guard(g.lock);
			t_lock.reset();
			B200Timer timer(B200_T_KERNEL_CALL);
			rc = b200_agg_sink(g.agg, batch, key_cols.data(), input_cols.empty() ? nullptr : input_cols.data());
		}
		b200_batch_free(batch); // b200_agg_sink returns after its kernels have read the batch
		B200Check(rc);
	}

	SinkResultType Sink(ExecutionContext &context, DataChunk &chunk, OperatorSinkInput &input) const override {
		auto &l = input.local_state.Cast<B200AggLocalState>();
		if (!on_device) {
			OperatorSinkInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Sink(context, chunk, inner_input);
		}
		auto &g = input.global_state.Cast<B200AggGlobalState>();
		idx_t from = 0;
		while (from < chunk.size()) {
			idx_t count = MinValue<idx_t>(chunk.size() - from, l.staging.Room());
			l.staging.Append(chunk, from, count);
			from += count;
			if (l.staging.Room() == 0) {
				// the morsel uploaded while this one was being filled is consumed now; then this one starts its upload
				SinkBatch(context, g, l.staging.TakeUploaded());
				l.staging.SubmitActive();
			}
		}
		return SinkResultType::NEED_MORE_INPUT;
	}

	SinkCombineResultType Combine(ExecutionContext &context, OperatorSinkCombineInput &input) const override {
		auto &l = input.local_state.Cast<B200AggLocalState>();
		if (!on_device) {
			OperatorSinkCombineInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Combine(context, inner_input);
		}
		auto &g = input.global_state.Cast<B200AggGlobalState>();
		SinkBatch(context, g, l.staging.TakeUploaded());
		l.staging.SubmitActive();
		SinkBatch(context, g, l.staging.TakeUploaded());
		return SinkCombineResultType::FINISHED;
	}

	SinkFinalizeType Finalize(Pipeline &pipeline, Event &event, ClientContext &context,
	                          OperatorSinkFinalizeInput &input) const override {
		if (!on_device) {
			OperatorSinkFinalizeInput inner_input {*inner.sink_state, input.interrupt_state};
			return inner.Finalize(pipeline, event, context, inner_input);
		}
		auto &g = input.global_state.Cast<B200AggGlobalState>();
		B200Timer timer(B200_T_FINALIZE);
		b200_batch *out = nullptr;
		B200Check(b200_agg_finalize(g.agg, &out));
		g.result_rows = b200_batch_rows(out);
		int ncols = b200_batch_cols(out);
		g.result_data.resize(ncols);
		g.result_valid.resize(ncols);
		for (int c = 0; c < ncols; c++) {
			b200_vector info;
			B200Check(b200_batch_column(out, c, &info));
			idx_t width = info.type == B200_INT128 ? 16 : GetTypeIdSize(static_cast<PhysicalType>(info.type));
			g.result_data[c].resize(g.result_rows * width + 16);
			g.result_valid[c].assign((g.result_rows + 63) / 64 + 1, 0);
			B200Check(b200_batch_download(g.ctx, out, c, g.result_data[c].data(), g.result_valid[c].data()));
		}
		b200_batch_free(out);
		g.finalized = true;
		return g.result_rows ? SinkFinalizeType::READY : SinkFinalizeType::NO_OUTPUT_POSSIBLE;
	}

	// ------------------------------------------------------------------ source
	bool IsSource() const override {
		return true;
	}
	bool ParallelSource() const override {
		return !on_device;
	}
	OrderPreservationType SourceOrder() const override {
		return OrderPreservationType::NO_ORDER;
	}

	unique_ptr<GlobalSourceState> GetGlobalSourceState(ClientContext &context) const override {
		auto state = make_uniq<B200AggSourceState>();
		if (!on_device) {
			state->inner = inner.GetGlobalSourceState(context);
		}
		return std::move(state);
	}
	unique_ptr<LocalSourceState> GetLocalSourceState(ExecutionContext &context, GlobalSourceState &gstate) const override {
		auto state = make_uniq<B200AggLocalSourceState>();
		if (!on_device) {
			state->inner = inner.GetLocalSourceState(context, *gstate.Cast<B200AggSourceState>().inner);
		}
		return std::move(state);
	}

	SourceResultType GetDataInternal(ExecutionContext &context, DataChunk &chunk,
	                                 OperatorSourceInput &input) const override {
		auto &src = input.global_state.Cast<B200AggSourceState>();
		if (!on_device) {
			OperatorSourceInput inner_input {*src.inner, *input.local_state.Cast<B200AggLocalSourceState>().inner,
			                                 input.interrupt_state};
			return inner.GetDataInternal(context, chunk, inner_input);
		}
		auto &g = sink_state->Cast<B200AggGlobalState>();
		if (src.position >= g.result_rows) {
			return SourceResultType::FINISHED;
		}
		idx_t count = MinValue<idx_t>(STANDARD_VECTOR_SIZE, g.result_rows - src.position);
		idx_t base = src.position;
		auto valid_at = [&](idx_t col, idx_t row) { return (g.result_valid[col][row >> 6] >> (row & 63)) & 1; };
		// output layout: [group columns, aggregate results] (radix_partitioned_hashtable.cpp:1341-1358)
		idx_t ngroups = plan.groups.size();
		for (idx_t c = 0; c < ngroups; c++) {
			auto &vec = chunk.data[c];
			idx_t width = plan.groups[c].width;
			memcpy(FlatVector::GetDataMutable(vec), g.result_data[c].data() + base * width, count * width);
			for (idx_t i = 0; i < count; i++) {
				if (!valid_at(c, base + i)) {
					FlatVector::SetNull(vec, i, true);
				}
			}
		}
		for (idx_t a = 0; a < plan.results.size(); a++) {
			auto &vec = chunk.data[ngroups + a];
			auto &res = plan.results[a];
			idx_t col = ngroups + res.desc;
			auto physical = vec.GetType().InternalType();
			for (idx_t i = 0; i < count; i++) {
				idx_t row = base + i;
				if (!valid_at(col, row)) {
					FlatVector::SetNull(vec, i, true);
					continue;
				}
				switch (res.kind) {
				case B200AggResult::DIRECT: {
					idx_t width = GetTypeIdSize(physical);
					memcpy(FlatVector::GetDataMutable(vec) + i * width, g.result_data[col].data() + row * width, width);
					break;
				}
				case B200AggResult::INT128_TO_RESULT: {
					auto src128 = reinterpret_cast<const hugeint_t *>(g.result_data[col].data()) + row;
					if (physical == PhysicalType::INT128) {
						FlatVector::GetDataMutableUnsafe<hugeint_t>(vec)[i] = *src128;
					} else {
						FlatVector::GetDataMutableUnsafe<int64_t>(vec)[i] = static_cast<int64_t>(src128->lower);
					}
					break;
				}
				case B200AggResult::AVG_INT: {
					auto sum = reinterpret_cast<const hugeint_t *>(g.result_data[col].data())[row];
					auto cnt = reinterpret_cast<const int64_t *>(g.result_data[col + 1].data())[row];
					if (cnt == 0) {
						FlatVector::SetNull(vec, i, true);
					} else if (res.int16) {
						// one rounding, as the stock operator: dividing in long double first would round twice
						FlatVector::GetDataMutableUnsafe<double>(vec)[i] =
						    Hugeint::Cast<double>(sum) / (static_cast<double>(cnt) * res.scale);
					} else {
						long double divident = static_cast<long double>(cnt) * static_cast<long double>(res.scale);
						FlatVector::GetDataMutableUnsafe<double>(vec)[i] =
						    static_cast<double>(Hugeint::Cast<long double>(sum) / divident);
					}
					break;
				}
				}
			}
		}
		chunk.SetCardinality(count);
		src.position += count;
		return SourceResultType::HAVE_MORE_OUTPUT;
	}
};

} // namespace duckdb
