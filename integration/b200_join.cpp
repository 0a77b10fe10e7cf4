#include <algorithm>
// Reference-side binding of the hash join (see INTEGRATION.md): B200HashJoin, a sink (build side) + operator
// (probe side) that DECORATES the stock PhysicalHashJoin the reference's planner produced.
//
//   replaces PhysicalHashJoin::{Sink,Combine,Finalize,ExecuteInternal}
//            (src/execution/operator/join/physical_hash_join.cpp:764,840,1893,2139)
//
// Eligible shapes: INNER / LEFT / SEMI / ANTI, equality conditions on BOUND_REF keys of numeric physical types,
// no residual predicate, build-side output columns of numeric physical types.  Probe-side output columns may have
// ANY type: the kernel returns the probe row id of every result row and the operator slices the input chunk with
// it (the same contract as ScanStructure::NextInnerJoin, join_hashtable.cpp:1737-1760).
// With a CUDA device: Sink batches build chunks into morsels -> b200_join_build_sink, Finalize ->
// b200_join_finalize, Execute -> b200_join_probe per input chunk, results emitted in <= 2048-row slices
// (HAVE_MORE_OUTPUT).  Without a device ("plumbing, no GPU") every call is forwarded to the wrapped operator.
#include "duckdb/execution/operator/join/physical_hash_join.hpp"
#include "duckdb/parallel/meta_pipeline.hpp"
#include "duckdb/parallel/pipeline.hpp"

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
	case JoinType::SEMI:
	case JoinType::ANTI:
		plan.join_type = static_cast<int32_t>(op.join_type); // b200_join_type uses duckdb::JoinType's values
		break;
	default:
		return plan;
	}
	if (op.predicate || op.residual_info || !op.delim_types.empty() || op.conditions.empty() ||
	    op.conditions.size() > 8) {
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
	bool with_payload = op.join_type == JoinType::INNER || op.join_type == JoinType::LEFT;
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
	if (op.types.size() != plan.lhs_output.size() + plan.payload.size()) {
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

class B200JoinLocalState : public LocalSinkState {
public:
	B200Morsel morsel;
	unique_ptr<LocalSinkState> inner;
};

//! Probe-side state of one worker: input chunks are buffered (deep copies + their key columns in a pinned staging
//! buffer) until a batch of B200_PROBE_BATCH rows is full, ONE b200_join_probe call handles the batch, and the result
//! rows are emitted chunk by chunk (HAVE_MORE_OUTPUT, then FinalExecute for the tail).  A per-chunk probe would be
//! one synchronous H2D -> kernel -> D2H round trip per 2048 rows.
class B200JoinOperatorState : public OperatorState {
public:
	unique_ptr<OperatorState> inner; // host mode
	// device mode
	B200Staging staging;                       // key columns of the buffered rows (pinned, uploaded on this worker's stream)
	vector<unique_ptr<DataChunk>> buffered;    // copies of the buffered input chunks (their vectors back the output slices)
	vector<idx_t> chunk_start;                 // first batch row of every buffered chunk
	idx_t buffered_rows = 0;
	bool input_taken = false;                  // the current input chunk is already in the buffer
	// results of the last probed batch, grouped by input chunk
	bool draining = false;
	vector<uint32_t> row_ids;                  // batch row of every result row, as returned
	vector<uint32_t> row_chunk;                // buffered chunk of every batch row
	vector<uint32_t> order;                    // result rows ordered by input chunk
	vector<idx_t> chunk_results;               // prefix: results of chunk c are order[chunk_results[c] .. chunk_results[c+1])
	idx_t emit_chunk = 0, emit_pos = 0;
	vector<vector<data_t>> payload_data;
	vector<vector<uint64_t>> payload_valid;
	uint32_t *sel_dev = nullptr;               // device buffer for the probe row id of every result row
	idx_t sel_capacity = 0;

	~B200JoinOperatorState() override {
		if (sel_dev) {
			cudaFree(sel_dev);
		}
	}
	void Finalize(const PhysicalOperator &op, ExecutionContext &context) override;
};

static constexpr idx_t B200_PROBE_BATCH = 128 * 1024;

class B200JoinSourceState : public GlobalSourceState {
public:
	unique_ptr<GlobalSourceState> inner;
	idx_t MaxThreads() override {
		return inner ? inner->MaxThreads() : 1;
	}
};

class B200JoinLocalSourceState : public LocalSourceState {
public:
	unique_ptr<LocalSourceState> inner;
};

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
		auto state = make_uniq<B200JoinLocalState>();
		if (!on_device) {
			state->inner = inner.GetLocalSinkState(context);
		} else {
			state->morsel.Init(plan.build_keys.size() + plan.payload.size());
		}
		return std::move(state);
	}

	void FlushBuild(B200JoinGlobalState &g, B200Morsel &m) const {
		if (m.rows == 0) {
			return;
		}
		vector<B200Column> infos = plan.build_keys;
		infos.insert(infos.end(), plan.payload.begin(), plan.payload.end());
		vector<b200_vector> cols;
		vector<vector<uint64_t>> masks;
		m.ToVectors(infos, cols, masks);
		vector<int> key_cols, payload_cols;
		for (idx_t c = 0; c < infos.size(); c++) {
			(c < plan.build_keys.size() ? key_cols : payload_cols).push_back(NumericCast<int>(c));
		}
		{
			std::lock_guard<std::mutex> guard(g.lock);
			B200Timer timer(B200_T_FINALIZE); // build side: upload + b200_join_build_sink
			b200_batch *batch = nullptr;
			B200Check(b200_batch_upload(g.ctx, cols.data(), NumericCast<int>(cols.size()), m.rows, &batch));
			int rc = b200_join_build_sink(g.join, batch, key_cols.data(), payload_cols.empty() ? nullptr : payload_cols.data());
			b200_ctx_sync(g.ctx);
			b200_batch_free(batch);
			B200Check(rc);
		}
		m.Clear();
	}

	SinkResultType Sink(ExecutionContext &context, DataChunk &chunk, OperatorSinkInput &input) const override {
		auto &l = input.local_state.Cast<B200JoinLocalState>();
		if (!on_device) {
			OperatorSinkInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Sink(context, chunk, inner_input);
		}
		idx_t c = 0;
		for (auto &k : plan.build_keys) {
			l.morsel.Append(chunk.data[k.chunk_col], c++, chunk.size(), k.width);
		}
		for (auto &p : plan.payload) {
			l.morsel.Append(chunk.data[p.chunk_col], c++, chunk.size(), p.width);
		}
		l.morsel.rows += chunk.size();
		if (l.morsel.rows >= B200_MORSEL_ROWS) {
			FlushBuild(input.global_state.Cast<B200JoinGlobalState>(), l.morsel);
		}
		return SinkResultType::NEED_MORE_INPUT;
	}

	SinkCombineResultType Combine(ExecutionContext &context, OperatorSinkCombineInput &input) const override {
		auto &l = input.local_state.Cast<B200JoinLocalState>();
		if (!on_device) {
			OperatorSinkCombineInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Combine(context, inner_input);
		}
		FlushBuild(input.global_state.Cast<B200JoinGlobalState>(), l.morsel);
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

	//! keep a copy of the input chunk and stage its key columns
	void BufferInput(ExecutionContext &context, B200JoinOperatorState &state, DataChunk &input) const {
		if (input.size() == 0) {
			return;
		}
		auto copy = make_uniq<DataChunk>();
		{
			B200Timer timer(B200_T_COPY_CHUNK);
			copy->Initialize(Allocator::Get(context.client), input.GetTypes());
			input.Copy(*copy);
		}
		state.staging.Append(*copy, 0, copy->size());
		state.chunk_start.push_back(state.buffered_rows);
		state.buffered_rows += copy->size();
		state.buffered.push_back(std::move(copy));
	}

	//! probe everything buffered with ONE kernel call; group the result rows by input chunk
	void ProbeBatch(ExecutionContext &context, B200JoinGlobalState &g, B200JoinOperatorState &state) const {
		context.client.InterruptCheck();
		state.draining = true;
		state.emit_chunk = 0;
		state.emit_pos = 0;
		idx_t n = state.buffered_rows;
		state.chunk_results.assign(state.buffered.size() + 1, 0);
		state.order.clear();
		if (n == 0) {
			return;
		}
		state.staging.SubmitActive();                   // H2D of the key columns on this worker's stream
		b200_batch *batch = state.staging.TakeUploaded(); // ... and wait for it (only this worker blocks)
		vector<int> key_cols;
		for (idx_t k = 0; k < plan.probe_keys.size(); k++) {
			key_cols.push_back(NumericCast<int>(k));
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
			auto ensure_sel = [&](uint64_t rows) {
				if (state.sel_capacity >= rows) {
					return true;
				}
				if (state.sel_dev) {
					cudaFree(state.sel_dev);
					state.sel_dev = nullptr;
				}
				state.sel_capacity = rows + rows / 4 + 1024;
				return cudaMalloc(reinterpret_cast<void **>(&state.sel_dev), state.sel_capacity * sizeof(uint32_t)) == cudaSuccess;
			};
			if (!ensure_sel(n)) {
				b200_batch_free(batch);
				throw OutOfMemoryException("b200: cannot allocate the probe selection buffer");
			}
			rc = b200_join_probe(g.join, batch, key_cols.data(), key_cols.data(), 0, n, &out, state.sel_dev, &count);
			if (rc == B200_ERR_CAPACITY) {
				rc = b200_join_probe(g.join, batch, key_cols.data(), key_cols.data(), 0, 0, &out, nullptr, &count);
				if (rc == B200_OK) {
					b200_batch_free(out);
					out = nullptr;
					if (!ensure_sel(count)) {
						b200_batch_free(batch);
						throw OutOfMemoryException("b200: cannot allocate the probe selection buffer");
					}
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

	//! emit the next <= 2048 result rows; returns false when the batch is drained (buffers are released)
	bool EmitNext(B200JoinOperatorState &state, DataChunk &chunk) const {
		B200Timer timer(B200_T_EMIT);
		while (state.emit_chunk < state.buffered.size() &&
		       state.chunk_results[state.emit_chunk] + state.emit_pos >= state.chunk_results[state.emit_chunk + 1]) {
			state.emit_chunk++;
			state.emit_pos = 0;
		}
		if (state.emit_chunk >= state.buffered.size()) {
			state.buffered.clear();
			state.chunk_start.clear();
			state.buffered_rows = 0;
			state.draining = false;
			chunk.SetCardinality(0);
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
		if (!state.input_taken) {
			BufferInput(context, state, input);
			state.input_taken = true;
			if (state.buffered_rows >= B200_PROBE_BATCH) {
				ProbeBatch(context, g, state);
			}
		}
		if (state.draining && EmitNext(state, chunk)) {
			return OperatorResultType::HAVE_MORE_OUTPUT; // called again with the same input (already buffered)
		}
		state.input_taken = false;
		return OperatorResultType::NEED_MORE_INPUT;
	}

	OperatorFinalizeResultType FinalExecute(ExecutionContext &context, DataChunk &chunk, GlobalOperatorState &gstate,
	                                        OperatorState &state_p) const override {
		auto &state = state_p.Cast<B200JoinOperatorState>();
		if (!on_device) {
			return inner.FinalExecute(context, chunk, gstate, *state.inner);
		}
		auto &g = sink_state->Cast<B200JoinGlobalState>();
		if (!state.draining && state.buffered_rows > 0) {
			ProbeBatch(context, g, state);
		}
		if (state.draining && EmitNext(state, chunk)) {
			return OperatorFinalizeResultType::HAVE_MORE_OUTPUT;
		}
		return OperatorFinalizeResultType::FINISHED;
	}

	// ------------------------------------------------------------------ source (host mode: external hash join)
	bool IsSource() const override {
		return on_device ? false : inner.IsSource();
	}
	bool ParallelSource() const override {
		return !on_device;
	}

	unique_ptr<GlobalSourceState> GetGlobalSourceState(ClientContext &context) const override {
		auto state = make_uniq<B200JoinSourceState>();
		if (!on_device) {
			state->inner = inner.GetGlobalSourceState(context);
		}
		return std::move(state);
	}
	unique_ptr<LocalSourceState> GetLocalSourceState(ExecutionContext &context, GlobalSourceState &gstate) const override {
		auto state = make_uniq<B200JoinLocalSourceState>();
		if (!on_device) {
			state->inner = inner.GetLocalSourceState(context, *gstate.Cast<B200JoinSourceState>().inner);
		}
		return std::move(state);
	}
	SourceResultType GetDataInternal(ExecutionContext &context, DataChunk &chunk,
	                                 OperatorSourceInput &input) const override {
		if (on_device) {
			return SourceResultType::FINISHED;
		}
		OperatorSourceInput inner_input {*input.global_state.Cast<B200JoinSourceState>().inner,
		                                 *input.local_state.Cast<B200JoinLocalSourceState>().inner, input.interrupt_state};
		return inner.GetData(context, chunk, inner_input);
	}
};

void B200JoinOperatorState::Finalize(const PhysicalOperator &op, ExecutionContext &context) {
	if (inner) {
		inner->Finalize(static_cast<const B200HashJoin &>(op).inner, context);
	}
}

} // namespace duckdb
