// Reference-side binding of the hash join (see INTEGRATION.md): B200HashJoin, a sink (build side) + operator
// (probe side) that DECORATES the stock PhysicalHashJoin the reference's planner produced.
//
//   replaces PhysicalHashJoin::{Sink,Combine,Finalize,ExecuteInternal}
//            (src/execution/operator/join/physical_hash_join.cpp:764,840,1893,2139)
//
// Eligible shapes: INNER / LEFT / RIGHT / FULL OUTER / SEMI / ANTI, equality conditions on BOUND_REF keys of numeric physical types,
// no residual predicate, build-side output columns of numeric physical types.  Probe-side output columns may have
// ANY type: the kernel returns the probe row id of every result row and the operator slices the input chunk with
// it (the same contract as ScanStructure::NextInnerJoin, join_hashtable.cpp:1737-1760).
// RIGHT and FULL OUTER joins probe like INNER and LEFT; the library flags every build row a probe emits.  Once every
// probe has run, the operator is also a source: workers take 1 Mi-row build ranges and emit the unflagged rows of each
// (b200_join_scan_unmatched) with NULL probe-side columns (JoinHashTable::ScanFullOuter, join_hashtable.cpp:2302-2356).
// MARK joins (large IN lists, IN subqueries that are not plain conjuncts) with ONE such condition, uncorrelated,
// without build-side output columns: the result is every probe row plus a BOOL mark, in probe order
// (b200_join_probe_mark), so each buffered input chunk is emitted whole with the mark vector appended.  Several
// conditions are left to the stock operator, whose row-equality MARK join compares NULL components row by row
// (JoinHashTable::InitializeUncorrelatedMarkJoin, physical_hash_join.cpp:710-720).
// With a CUDA device: Sink streams build chunks through the worker's staging ring -> b200_join_build_sink per
// morsel, Finalize -> b200_join_finalize, Execute -> b200_join_probe per batch of buffered input chunks, results
// emitted in <= 2048-row slices (HAVE_MORE_OUTPUT).  Without a device ("plumbing, no GPU") every call is forwarded to
// the wrapped operator.
#include "b200_binding.hpp"

#include "duckdb/common/vector/constant_vector.hpp"
#include "duckdb/common/vector/flat_vector.hpp"
#include "duckdb/execution/operator/join/physical_hash_join.hpp"
#include "duckdb/parallel/meta_pipeline.hpp"
#include "duckdb/parallel/pipeline.hpp"
#include "duckdb/planner/expression/bound_reference_expression.hpp"

#include <algorithm>

namespace duckdb {

struct B200JoinPlan {
	bool eligible = false;
	int32_t join_type = 0;
	vector<B200Column> build_keys;
	vector<B200Column> probe_keys;
	vector<B200Column> payload;     // build-chunk columns behind rhs_output_columns, in output order
	vector<idx_t> lhs_output;       // probe-chunk columns, in output order
};

static B200JoinPlan AnalyseJoin(const PhysicalHashJoin &op) {
	B200JoinPlan plan;
	switch (op.join_type) {
	case JoinType::INNER:
	case JoinType::LEFT:
	case JoinType::RIGHT:
	case JoinType::OUTER:
	case JoinType::SEMI:
	case JoinType::ANTI:
	case JoinType::MARK:
		plan.join_type = static_cast<int32_t>(op.join_type); // b200_join_type uses duckdb::JoinType's values
		break;
	default:
		return plan;
	}
	bool mark = op.join_type == JoinType::MARK;
	if (op.predicate || op.residual_info || !op.delim_types.empty() || op.conditions.empty() ||
	    op.conditions.size() > (mark ? 1 : 8)) {
		return plan;
	}
	for (auto &cond : op.conditions) {
		if (!cond.IsComparison() || cond.GetComparisonType() != ExpressionType::COMPARE_EQUAL) {
			return plan;
		}
		auto &lhs = cond.GetLHS();
		auto &rhs = cond.GetRHS();
		int32_t ltype, rtype;
		if (lhs.GetExpressionClass() != ExpressionClass::BOUND_REF || rhs.GetExpressionClass() != ExpressionClass::BOUND_REF ||
		    !B200Type(lhs.GetReturnType().InternalType(), ltype) || !B200Type(rhs.GetReturnType().InternalType(), rtype) ||
		    ltype != rtype) {
			return plan;
		}
		idx_t width = GetTypeIdSize(lhs.GetReturnType().InternalType());
		plan.probe_keys.push_back({lhs.Cast<BoundReferenceExpression>().Index(), ltype, width});
		plan.build_keys.push_back({rhs.Cast<BoundReferenceExpression>().Index(), rtype, width});
	}
	bool with_payload = op.join_type == JoinType::INNER || op.join_type == JoinType::LEFT ||
	                    op.join_type == JoinType::RIGHT || op.join_type == JoinType::OUTER;
	if (with_payload) {
		// rhs_output_columns index the hash table layout [keys..., payload...] (physical_hash_join.cpp:209-232)
		idx_t nkeys = op.conditions.size();
		for (idx_t i = 0; i < op.rhs_output_columns.col_idxs.size(); i++) {
			idx_t layout_col = op.rhs_output_columns.col_idxs[i];
			idx_t chunk_col = layout_col < nkeys ? plan.build_keys[layout_col].chunk_col
			                                     : op.payload_columns.col_idxs[layout_col - nkeys];
			int32_t type;
			auto physical = op.rhs_output_columns.col_types[i].InternalType();
			if (!B200Type(physical, type)) {
				return plan;
			}
			plan.payload.push_back({chunk_col, type, GetTypeIdSize(physical)});
		}
		if (plan.payload.size() > 12) {
			return plan;
		}
	} else if (!op.rhs_output_columns.col_idxs.empty()) {
		return plan;
	}
	plan.lhs_output = op.lhs_output_columns.col_idxs;
	if (op.types.size() != plan.lhs_output.size() + plan.payload.size() + (mark ? 1 : 0) ||
	    (mark && op.types.back().id() != LogicalTypeId::BOOLEAN)) {
		return plan;
	}
	plan.eligible = true;
	return plan;
}

class B200JoinGlobalState : public GlobalSinkState {
public:
	std::mutex lock;
	b200_ctx *ctx = nullptr;
	b200_join *join = nullptr;

	~B200JoinGlobalState() override {
		B200TimingReport("hash join");
		if (join) {
			b200_join_destroy(join);
		}
		B200ContextPool::Release(ctx);
	}
};

//! Probe-side state of one worker: batches of B200_PROBE_BATCH rows (their key columns staged), ONE b200_join_probe
//! call per batch
class B200JoinOperatorState : public B200BatchState {
public:
	unique_ptr<OperatorState> inner; // host mode
	// results of the last probed batch, grouped by input chunk
	vector<uint32_t> row_ids;                  // batch row of every result row, as returned
	vector<uint32_t> row_chunk;                // buffered chunk of every batch row
	vector<uint32_t> order;                    // result rows ordered by input chunk
	vector<idx_t> chunk_results;               // prefix: results of chunk c are order[chunk_results[c] .. chunk_results[c+1])
	vector<vector<data_t>> payload_data;
	vector<vector<uint64_t>> payload_valid;
	// MARK join: one device block and its pinned host copy, [validity words | mark bytes] of the batch
	void *mark_dev = nullptr;
	uint8_t *mark_host = nullptr;

	~B200JoinOperatorState() override {
		if (mark_dev) {
			cudaFree(mark_dev);
		}
		if (mark_host) {
			b200_host_free(nullptr, mark_host);
		}
	}
	void Finalize(const PhysicalOperator &op, ExecutionContext &context) override;
};

static constexpr idx_t B200_PROBE_BATCH = 128 * 1024;
//! RIGHT / FULL OUTER source phase: build rows per b200_join_scan_unmatched call (a multiple of 64)
static constexpr idx_t B200_SCAN_RANGE = 1 << 20;

//! RIGHT / FULL OUTER source phase: the next build range to scan
class B200JoinSourceState : public B200SourceState {
public:
	std::atomic<idx_t> next_range {0};
	idx_t ranges = 0;
	idx_t MaxThreads() override {
		return inner ? inner->MaxThreads() : MaxValue<idx_t>(ranges, 1);
	}
};

//! RIGHT / FULL OUTER source phase: the unmatched build rows of the worker's current range, on the host
class B200JoinLocalSourceState : public B200LocalSourceState {
public:
	vector<vector<data_t>> payload_data;
	vector<vector<uint64_t>> payload_valid;
	idx_t count = 0;
	idx_t emitted = 0;
};
//! MARK join block: validity words, then mark bytes, for a batch of at most one chunk past B200_PROBE_BATCH rows
static constexpr idx_t B200_MARK_ROWS = B200_PROBE_BATCH + STANDARD_VECTOR_SIZE;
static constexpr idx_t B200_MARK_VALID_BYTES = (B200_MARK_ROWS + 63) / 64 * 8;

class B200HashJoin : public PhysicalOperator {
public:
	B200HashJoin(PhysicalPlan &physical_plan, PhysicalHashJoin &inner_p, B200JoinPlan plan_p)
	    : PhysicalOperator(physical_plan, PhysicalOperatorType::EXTENSION, inner_p.types, inner_p.estimated_cardinality),
	      inner(inner_p), plan(std::move(plan_p)), on_device(b200_device_count() > 0) {
		for (auto &child : inner_p.children) {
			children.push_back(child);
		}
	}

	//! the stock operator this one decorates (same plan arena); the base-class view reaches the interface methods
	//! PhysicalHashJoin re-declares as protected
	PhysicalOperator &inner;
	B200JoinPlan plan;
	bool on_device;

	string GetName() const override {
		return on_device ? "B200_HASH_JOIN" : "B200_HASH_JOIN(host)";
	}
	InsertionOrderPreservingMap<string> ParamsToString() const override {
		auto result = inner.ParamsToString();
		result["Operator"] = GetName();
		return result;
	}

	// ------------------------------------------------------------------ pipelines
	// Same shape as PhysicalJoin::BuildJoinPipelines (physical_join.cpp:31-83): this operator joins the probe
	// pipeline, its build side becomes a child meta-pipeline with this operator as the sink.
	void BuildPipelines(Pipeline &current, MetaPipeline &meta_pipeline) override {
		op_state.reset();
		sink_state.reset();
		meta_pipeline.GetState().AddPipelineOperator(current, *this);

		vector<shared_ptr<Pipeline>> before;
		meta_pipeline.GetPipelines(before, false);
		auto &last_pipeline = *before.back();

		auto &build_side = meta_pipeline.CreateChildMetaPipeline(current, *this, MetaPipelineType::JOIN_BUILD);
		build_side.Build(children[1]);
		vector<shared_ptr<Pipeline>> dependencies;
		optional_ptr<MetaPipeline> last_child;
		if (children[1].get().CanSaturateThreads(current.GetClientContext())) {
			build_side.GetPipelines(dependencies, false);
			last_child = meta_pipeline.GetLastChild();
		}
		children[0].get().BuildPipelines(current, meta_pipeline);
		if (last_child) {
			meta_pipeline.AddRecursiveDependencies(dependencies, *last_child);
		}
		if (IsSource()) {
			meta_pipeline.CreateChildPipeline(current, *this, last_pipeline);
		}
	}

	vector<const_reference<PhysicalOperator>> GetSources() const override {
		auto result = children[0].get().GetSources();
		if (IsSource()) {
			result.push_back(*this);
		}
		return result;
	}

	// ------------------------------------------------------------------ sink (build side)
	bool IsSink() const override {
		return true;
	}
	bool ParallelSink() const override {
		return true;
	}

	unique_ptr<GlobalSinkState> GetGlobalSinkState(ClientContext &context) const override {
		auto state = make_uniq<B200JoinGlobalState>();
		if (!on_device) {
			inner.sink_state = inner.GetGlobalSinkState(context);
			return std::move(state);
		}
		state->ctx = B200ContextPool::Acquire(0);
		vector<int32_t> key_types, payload_types;
		for (auto &k : plan.build_keys) {
			key_types.push_back(k.type);
		}
		for (auto &p : plan.payload) {
			payload_types.push_back(p.type);
		}
		B200Check(b200_join_create(state->ctx, plan.join_type, key_types.data(), NumericCast<int>(key_types.size()),
		                           payload_types.empty() ? nullptr : payload_types.data(),
		                           NumericCast<int>(payload_types.size()), &state->join));
		return std::move(state);
	}

	unique_ptr<LocalSinkState> GetLocalSinkState(ExecutionContext &context) const override {
		auto state = make_uniq<B200LocalSinkState>();
		if (!on_device) {
			state->inner = inner.GetLocalSinkState(context);
		} else {
			vector<B200Column> infos = plan.build_keys;
			infos.insert(infos.end(), plan.payload.begin(), plan.payload.end());
			state->staging.Init(0, infos, B200_MORSEL_ROWS);
		}
		return std::move(state);
	}

	//! sink one uploaded morsel of build rows: the join object lives on the global context and is driven by one thread
	//! at a time
	void SinkBuildBatch(B200JoinGlobalState &g, b200_batch *batch) const {
		if (!batch) {
			return;
		}
		vector<int> key_cols, payload_cols;
		for (idx_t c = 0; c < plan.build_keys.size() + plan.payload.size(); c++) {
			(c < plan.build_keys.size() ? key_cols : payload_cols).push_back(NumericCast<int>(c));
		}
		int rc;
		{
			auto t_lock = make_uniq<B200Timer>(B200_T_LOCK_WAIT);
			std::lock_guard<std::mutex> guard(g.lock);
			t_lock.reset();
			B200Timer timer(B200_T_KERNEL_CALL);
			rc = b200_join_build_sink(g.join, batch, key_cols.data(), payload_cols.empty() ? nullptr : payload_cols.data());
			// the build kernels read the worker's ring buffer asynchronously on the join's stream, and the ring refills
			// that buffer two morsels later
			b200_ctx_sync(g.ctx);
		}
		b200_batch_free(batch);
		B200Check(rc);
	}

	SinkResultType Sink(ExecutionContext &context, DataChunk &chunk, OperatorSinkInput &input) const override {
		auto &l = input.local_state.Cast<B200LocalSinkState>();
		if (!on_device) {
			OperatorSinkInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Sink(context, chunk, inner_input);
		}
		auto &g = input.global_state.Cast<B200JoinGlobalState>();
		l.staging.Feed(chunk, [&](b200_batch *batch) { SinkBuildBatch(g, batch); });
		return SinkResultType::NEED_MORE_INPUT;
	}

	SinkCombineResultType Combine(ExecutionContext &context, OperatorSinkCombineInput &input) const override {
		auto &l = input.local_state.Cast<B200LocalSinkState>();
		if (!on_device) {
			OperatorSinkCombineInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Combine(context, inner_input);
		}
		auto &g = input.global_state.Cast<B200JoinGlobalState>();
		l.staging.Drain([&](b200_batch *batch) { SinkBuildBatch(g, batch); });
		return SinkCombineResultType::FINISHED;
	}

	void PrepareFinalize(ClientContext &context, GlobalSinkState &state) const override {
		if (!on_device) {
			inner.PrepareFinalize(context, *inner.sink_state);
		}
	}

	SinkFinalizeType Finalize(Pipeline &pipeline, Event &event, ClientContext &context,
	                          OperatorSinkFinalizeInput &input) const override {
		if (!on_device) {
			OperatorSinkFinalizeInput inner_input {*inner.sink_state, input.interrupt_state};
			return inner.Finalize(pipeline, event, context, inner_input);
		}
		auto &g = input.global_state.Cast<B200JoinGlobalState>();
		B200Check(b200_join_finalize(g.join));
		return SinkFinalizeType::READY;
	}

	// ------------------------------------------------------------------ operator (probe side)
	bool ParallelOperator() const override {
		return true;
	}
	bool RequiresFinalExecute() const override {
		return on_device ? true : inner.RequiresFinalExecute(); // device mode: the last, partial batch is probed at the end
	}

	unique_ptr<OperatorState> GetOperatorState(ExecutionContext &context) const override {
		auto state = make_uniq<B200JoinOperatorState>();
		if (!on_device) {
			state->inner = inner.GetOperatorState(context);
		} else {
			state->staging.Init(0, plan.probe_keys, B200_PROBE_BATCH + STANDARD_VECTOR_SIZE);
			state->payload_data.resize(plan.payload.size());
			state->payload_valid.resize(plan.payload.size());
		}
		return std::move(state);
	}

	//! probe everything buffered with ONE kernel call; group the result rows by input chunk
	void ProbeBatch(B200JoinGlobalState &g, B200JoinOperatorState &state, b200_batch *batch) const {
		idx_t n = state.buffered_rows;
		state.chunk_results.assign(state.buffered.size() + 1, 0);
		state.order.clear();
		vector<int> key_cols;
		for (idx_t k = 0; k < plan.probe_keys.size(); k++) {
			key_cols.push_back(NumericCast<int>(k));
		}
		if (plan.join_type == B200_JOIN_MARK) {
			ProbeMarkBatch(g, state, batch, key_cols);
			return;
		}
		// result rows <= probe rows x longest duplicate chain; sized by the library (capacity 0) except for the row ids
		b200_batch *out = nullptr;
		uint64_t count = 0;
		int rc;
		{
			auto t_lock = make_uniq<B200Timer>(B200_T_LOCK_WAIT);
			std::lock_guard<std::mutex> guard(g.lock); // one join object (one stream), driven from one thread at a time
			t_lock.reset();
			B200Timer timer(B200_T_KERNEL_CALL);
			// one pass when the result fits n rows (always, for a unique build key: PK-FK joins); duplicates on the build
			// side can produce more rows than probes: then a counting call sizes the second attempt exactly
			state.ReserveSel(n, batch);
			rc = b200_join_probe(g.join, batch, key_cols.data(), key_cols.data(), 0, n, &out, state.sel_dev, &count);
			if (rc == B200_ERR_CAPACITY) {
				rc = b200_join_probe(g.join, batch, key_cols.data(), key_cols.data(), 0, 0, &out, nullptr, &count);
				if (rc == B200_OK) {
					b200_batch_free(out);
					out = nullptr;
					state.ReserveSel(count, batch);
					rc = b200_join_probe(g.join, batch, key_cols.data(), key_cols.data(), 0, count, &out, state.sel_dev, &count);
				}
			}
			b200_batch_free(batch);
			B200Check(rc);
			state.row_ids.resize(count + 1);
			if (count > 0) {
				if (cudaMemcpy(state.row_ids.data(), state.sel_dev, count * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) {
					b200_batch_free(out);
					throw IOException("b200: D2H of the probe row ids failed");
				}
			}
			for (idx_t p = 0; p < plan.payload.size() && rc == B200_OK; p++) {
				state.payload_data[p].resize(count * plan.payload[p].width + 16);
				state.payload_valid[p].assign((count + 63) / 64 + 1, 0);
				rc = b200_batch_download(g.ctx, out, NumericCast<int>(p), state.payload_data[p].data(),
				                         state.payload_valid[p].data());
			}
		}
		b200_batch_free(out);
		B200Check(rc);
		B200Timer timer_sort(B200_T_DOWNLOAD); // host-side grouping of the result rows
		// counting sort of the result rows by input chunk (an output chunk slices ONE input chunk)
		idx_t nchunks = state.buffered.size();
		// batch row -> buffered chunk, by table (chunks are <= 2048 rows but not all full)
		state.row_chunk.resize(n);
		for (idx_t c = 0; c < nchunks; c++) {
			idx_t end = c + 1 < nchunks ? state.chunk_start[c + 1] : n;
			std::fill(state.row_chunk.begin() + NumericCast<int64_t>(state.chunk_start[c]),
			          state.row_chunk.begin() + NumericCast<int64_t>(end), NumericCast<uint32_t>(c));
		}
		vector<uint32_t> chunk_of(count);
		for (idx_t i = 0; i < count; i++) {
			uint32_t c = state.row_chunk[state.row_ids[i]];
			chunk_of[i] = c;
			state.chunk_results[idx_t(c) + 1]++;
		}
		for (idx_t c = 0; c < nchunks; c++) {
			state.chunk_results[c + 1] += state.chunk_results[c];
		}
		state.order.resize(count);
		vector<idx_t> cursor(state.chunk_results.begin(), state.chunk_results.end() - 1);
		for (idx_t i = 0; i < count; i++) {
			state.order[cursor[chunk_of[i]]++] = NumericCast<uint32_t>(i);
		}
	}

	//! MARK join: one in-order kernel call for the batch, then ONE copy of its marks and validity to the host
	void ProbeMarkBatch(B200JoinGlobalState &g, B200JoinOperatorState &state, b200_batch *batch,
	                    const vector<int> &key_cols) const {
		int rc;
		{
			auto t_lock = make_uniq<B200Timer>(B200_T_LOCK_WAIT);
			std::lock_guard<std::mutex> guard(g.lock); // one join object (one stream), driven from one thread at a time
			t_lock.reset();
			B200Timer timer(B200_T_KERNEL_CALL);
			if (!state.mark_dev) {
				if (cudaMalloc(&state.mark_dev, B200_MARK_VALID_BYTES + B200_MARK_ROWS) != cudaSuccess ||
				    b200_host_alloc(g.ctx, B200_MARK_VALID_BYTES + B200_MARK_ROWS, reinterpret_cast<void **>(&state.mark_host)) != B200_OK) {
					b200_batch_free(batch);
					throw OutOfMemoryException("b200: cannot allocate the MARK join result buffers");
				}
			}
			auto block = static_cast<uint8_t *>(state.mark_dev);
			rc = b200_join_probe_mark(g.join, batch, key_cols.data(), block + B200_MARK_VALID_BYTES,
			                          reinterpret_cast<uint64_t *>(block));
			if (rc == B200_OK) {
				rc = b200_ctx_sync(g.ctx);
			}
			b200_batch_free(batch);
		}
		B200Check(rc);
		B200Timer timer(B200_T_DOWNLOAD);
		if (cudaMemcpy(state.mark_host, state.mark_dev, B200_MARK_VALID_BYTES + state.buffered_rows,
		               cudaMemcpyDeviceToHost) != cudaSuccess) {
			throw IOException("b200: D2H of the MARK join result failed");
		}
	}

	//! MARK join: the next buffered input chunk, whole, with its marks appended (ConstructMarkJoinResult's layout)
	bool EmitNextMark(B200JoinOperatorState &state, DataChunk &chunk) const {
		B200Timer timer(B200_T_EMIT);
		if (state.emit_chunk >= state.buffered.size()) {
			return false;
		}
		idx_t c = state.emit_chunk++;
		auto &src = *state.buffered[c];
		idx_t count = src.size();
		idx_t start = state.chunk_start[c];
		idx_t nlhs = plan.lhs_output.size();
		for (idx_t col = 0; col < nlhs; col++) {
			chunk.data[col].Reference(src.data[plan.lhs_output[col]]);
		}
		auto &mark = chunk.data[nlhs];
		mark.SetVectorType(VectorType::FLAT_VECTOR);
		FlatVector::SetSize(mark, count_t(count));
		chunk.SetChildCardinality(count); // after the references: a referenced constant vector is resized too
		auto out = FlatVector::GetDataMutable<bool>(mark);
		auto &mask = FlatVector::ValidityMutable(mark);
		mask.SetAllValid(count);
		auto valid = reinterpret_cast<const uint64_t *>(state.mark_host);
		const uint8_t *marks = state.mark_host + B200_MARK_VALID_BYTES + start;
		for (idx_t i = 0; i < count; i++) {
			out[i] = marks[i] != 0;
			idx_t row = start + i;
			if (!((valid[row >> 6] >> (row & 63)) & 1)) {
				mask.SetInvalid(i);
			}
		}
		return true;
	}

	//! emit the next <= 2048 result rows; returns false when the batch is drained
	bool EmitNext(B200JoinOperatorState &state, DataChunk &chunk) const {
		if (plan.join_type == B200_JOIN_MARK) {
			return EmitNextMark(state, chunk);
		}
		B200Timer timer(B200_T_EMIT);
		while (state.emit_chunk < state.buffered.size() &&
		       state.chunk_results[state.emit_chunk] + state.emit_pos >= state.chunk_results[state.emit_chunk + 1]) {
			state.emit_chunk++;
			state.emit_pos = 0;
		}
		if (state.emit_chunk >= state.buffered.size()) {
			return false;
		}
		idx_t c = state.emit_chunk;
		idx_t first = state.chunk_results[c] + state.emit_pos;
		idx_t count = MinValue<idx_t>(STANDARD_VECTOR_SIZE, state.chunk_results[c + 1] - first);
		auto &src = *state.buffered[c];
		// probe-side columns: slices of the buffered input chunk (any type), like chunk.Slice(left, sel, n)
		SelectionVector sel(STANDARD_VECTOR_SIZE);
		for (idx_t i = 0; i < count; i++) {
			sel.set_index(i, state.row_ids[state.order[first + i]] - state.chunk_start[c]);
		}
		idx_t nlhs = plan.lhs_output.size();
		for (idx_t col = 0; col < nlhs; col++) {
			chunk.data[col].Slice(src.data[plan.lhs_output[col]], sel, count);
		}
		// build-side columns: gathered by the kernel
		for (idx_t p = 0; p < plan.payload.size(); p++) {
			auto &vec = chunk.data[nlhs + p];
			idx_t width = plan.payload[p].width;
			auto dst = FlatVector::GetDataMutable(vec);
			auto &valid = state.payload_valid[p];
			auto src_data = state.payload_data[p].data();
			auto gather = [&](auto tag) {
				using T = decltype(tag);
				auto out = reinterpret_cast<T *>(dst);
				auto in = reinterpret_cast<const T *>(src_data);
				for (idx_t i = 0; i < count; i++) {
					out[i] = in[state.order[first + i]];
				}
			};
			switch (width) {
			case 1:
				gather(uint8_t(0));
				break;
			case 2:
				gather(uint16_t(0));
				break;
			case 4:
				gather(uint32_t(0));
				break;
			default:
				gather(uint64_t(0));
				break;
			}
			for (idx_t i = 0; i < count; i++) {
				idx_t row = state.order[first + i];
				if (!((valid[row >> 6] >> (row & 63)) & 1)) {
					FlatVector::SetNull(vec, i, true);
				}
			}
		}
		chunk.SetCardinality(count);
		state.emit_pos += count;
		return true;
	}

	OperatorResultType Execute(ExecutionContext &context, DataChunk &input, DataChunk &chunk,
	                           GlobalOperatorState &gstate, OperatorState &state_p) const override {
		auto &state = state_p.Cast<B200JoinOperatorState>();
		if (!on_device) {
			return inner.Execute(context, input, chunk, gstate, *state.inner);
		}
		auto &g = sink_state->Cast<B200JoinGlobalState>();
		return state.Execute(
		    context, input, chunk, B200_PROBE_BATCH, [&](b200_batch *batch) { ProbeBatch(g, state, batch); },
		    [&](DataChunk &out) { return EmitNext(state, out); });
	}

	OperatorFinalizeResultType FinalExecute(ExecutionContext &context, DataChunk &chunk, GlobalOperatorState &gstate,
	                                        OperatorState &state_p) const override {
		auto &state = state_p.Cast<B200JoinOperatorState>();
		if (!on_device) {
			return inner.FinalExecute(context, chunk, gstate, *state.inner);
		}
		auto &g = sink_state->Cast<B200JoinGlobalState>();
		return state.FinalExecute(
		    context, chunk, [&](b200_batch *batch) { ProbeBatch(g, state, batch); },
		    [&](DataChunk &out) { return EmitNext(state, out); });
	}

	// ------------------------------------------------------------------ source (host mode: external hash join)
	// ------------------------------------------------------------------ source (device: the unmatched build rows of
	// RIGHT / FULL OUTER joins; host mode: whatever the stock operator emits, e.g. its external hash join)
	bool EmitsBuildSide() const {
		return plan.join_type == B200_JOIN_RIGHT || plan.join_type == B200_JOIN_OUTER;
	}
	bool IsSource() const override {
		return on_device ? EmitsBuildSide() : inner.IsSource();
	}
	bool ParallelSource() const override {
		return !on_device || EmitsBuildSide();
	}

	unique_ptr<GlobalSourceState> GetGlobalSourceState(ClientContext &context) const override {
		auto state = make_uniq<B200JoinSourceState>();
		if (!on_device) {
			state->inner = inner.GetGlobalSourceState(context);
		} else if (sink_state) {
			uint64_t rows = 0;
			B200Check(b200_join_build_rows(sink_state->Cast<B200JoinGlobalState>().join, &rows));
			state->ranges = (rows + B200_SCAN_RANGE - 1) / B200_SCAN_RANGE;
		}
		return std::move(state);
	}
	unique_ptr<LocalSourceState> GetLocalSourceState(ExecutionContext &context, GlobalSourceState &gstate) const override {
		auto state = make_uniq<B200JoinLocalSourceState>();
		if (!on_device) {
			state->inner = inner.GetLocalSourceState(context, *gstate.Cast<B200SourceState>().inner);
		} else {
			state->payload_data.resize(plan.payload.size());
			state->payload_valid.resize(plan.payload.size());
		}
		return std::move(state);
	}

	//! scan the next build range of this worker into its host buffers; false when every range is taken
	bool ScanNextRange(B200JoinGlobalState &g, B200JoinSourceState &gs, B200JoinLocalSourceState &l) const {
		idx_t range = gs.next_range++;
		if (range >= gs.ranges) {
			return false;
		}
		b200_batch *out = nullptr;
		uint64_t count = 0;
		int rc;
		{
			auto t_lock = make_uniq<B200Timer>(B200_T_LOCK_WAIT);
			std::lock_guard<std::mutex> guard(g.lock); // one join object (one stream), driven from one thread at a time
			t_lock.reset();
			B200Timer timer(B200_T_KERNEL_CALL);
			uint64_t rows = 0;
			rc = b200_join_build_rows(g.join, &rows);
			uint64_t begin = range * B200_SCAN_RANGE;
			uint64_t end = MinValue<uint64_t>(begin + B200_SCAN_RANGE, rows);
			if (rc == B200_OK) {
				rc = b200_join_scan_unmatched(g.join, begin, end, &out, nullptr, &count);
			}
			for (idx_t p = 0; p < plan.payload.size() && rc == B200_OK; p++) {
				l.payload_data[p].resize(count * plan.payload[p].width + 16);
				l.payload_valid[p].assign((count + 63) / 64 + 1, 0);
				rc = b200_batch_download(g.ctx, out, NumericCast<int>(p), l.payload_data[p].data(),
				                         l.payload_valid[p].data());
			}
		}
		b200_batch_free(out);
		B200Check(rc);
		l.count = count;
		l.emitted = 0;
		return true;
	}

	//! the next <= 2048 unmatched build rows: constant NULL probe-side columns, the build columns copied as EmitNext
	//! copies them
	void EmitUnmatched(B200JoinLocalSourceState &l, DataChunk &chunk) const {
		B200Timer timer(B200_T_EMIT);
		idx_t first = l.emitted;
		idx_t count = MinValue<idx_t>(STANDARD_VECTOR_SIZE, l.count - first);
		idx_t nlhs = plan.lhs_output.size();
		for (idx_t col = 0; col < nlhs; col++) {
			chunk.data[col].SetVectorType(VectorType::CONSTANT_VECTOR);
			ConstantVector::SetNull(chunk.data[col], true);
		}
		for (idx_t p = 0; p < plan.payload.size(); p++) {
			auto &vec = chunk.data[nlhs + p];
			idx_t width = plan.payload[p].width;
			memcpy(FlatVector::GetDataMutable(vec), l.payload_data[p].data() + first * width, count * width);
			auto &valid = l.payload_valid[p];
			for (idx_t i = 0; i < count; i++) {
				idx_t row = first + i;
				if (!((valid[row >> 6] >> (row & 63)) & 1)) {
					FlatVector::SetNull(vec, i, true);
				}
			}
		}
		chunk.SetCardinality(count);
		l.emitted += count;
	}

	SourceResultType GetDataInternal(ExecutionContext &context, DataChunk &chunk,
	                                 OperatorSourceInput &input) const override {
		if (on_device) {
			auto &g = sink_state->Cast<B200JoinGlobalState>();
			auto &gs = input.global_state.Cast<B200JoinSourceState>();
			auto &l = input.local_state.Cast<B200JoinLocalSourceState>();
			while (l.emitted >= l.count) {
				if (!ScanNextRange(g, gs, l)) {
					return SourceResultType::FINISHED;
				}
			}
			EmitUnmatched(l, chunk);
			return SourceResultType::HAVE_MORE_OUTPUT;
		}
		OperatorSourceInput inner_input {*input.global_state.Cast<B200SourceState>().inner,
		                                 *input.local_state.Cast<B200LocalSourceState>().inner, input.interrupt_state};
		return inner.GetData(context, chunk, inner_input);
	}
};

void B200JoinOperatorState::Finalize(const PhysicalOperator &op, ExecutionContext &context) {
	if (inner) {
		inner->Finalize(static_cast<const B200HashJoin &>(op).inner, context);
	}
}

} // namespace duckdb
