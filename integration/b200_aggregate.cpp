// Reference-side binding of the hash aggregate (see INTEGRATION.md): B200HashAggregate, a sink + source
// PhysicalOperator that DECORATES the stock PhysicalHashAggregate the reference's planner produced.
//
//   replaces PhysicalHashAggregate::{Sink,Combine,Finalize,GetDataInternal}
//            (src/execution/operator/aggregate/physical_hash_aggregate.cpp:415,503,838,958)
//
// The stock operator is planned as usual (so groups / aggregates are already reduced to BOUND_REFs of the child
// chunk, plan_aggregate.cpp:313+); when its shape is eligible - one grouping set, no DISTINCT, group and aggregate
// inputs of numeric physical types, aggregates in {count_star, count, sum, sum_no_overflow, min, max, avg}, each
// with or without a FILTER - it is wrapped.  The planner has already moved every FILTER (WHERE ...) into the
// projection below as a BOOLEAN column (plan_aggregate.cpp:342-348), so a filter is one more staged column, and
// b200_agg_create_filtered applies it on the device (this is also what a small PIVOT binds to: one filtered
// aggregate per pivot value, bind_pivot.cpp:164-205).  With a CUDA device the wrapper batches the 2048-row chunks into morsels, uploads them
// and calls b200_agg_sink; Finalize downloads [groups..., results...] and GetData emits them in <= 2048-row
// chunks.  Without a device ("plumbing, no GPU") every call is forwarded to the wrapped stock operator.
// Ineligible aggregates are not wrapped at all (the plan keeps the stock operator).
#include "b200_binding.hpp"

#include "duckdb/execution/operator/aggregate/physical_hash_aggregate.hpp"
#include "duckdb/planner/expression/bound_aggregate_expression.hpp"
#include "duckdb/planner/expression/bound_reference_expression.hpp"
#include "duckdb/common/types/hugeint.hpp"
#include "duckdb/common/vector/flat_vector.hpp"

#include <algorithm>
#include <cmath>

namespace duckdb {

struct B200AggResult {
	enum Kind { DIRECT, INT128_TO_RESULT, AVG_INT } kind;
	int desc;       // index of the b200 aggregate (AVG_INT: the SUM, desc + 1 is the COUNT)
	double scale;   // AVG over DECIMAL: 10^scale, else 1
	bool int16;     // AVG_INT over an INT16 input (SMALLINT, DECIMAL(<=4)): divided in double, not long double
};

struct B200AggPlan {
	bool eligible = false;
	vector<B200Column> groups;
	vector<B200Column> inputs; // distinct chunk columns the aggregates read: inputs and BOOLEAN filter columns
	vector<b200_agg_desc> descs;
	vector<int32_t> filters; // per desc: -1, or the index in `inputs` of its filter column
	bool has_filter = false;
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
	// the staged column of chunk column `col` (one per chunk column, whatever reads it)
	auto staged = [&](idx_t col, int32_t type, idx_t width) {
		for (idx_t i = 0; i < plan.inputs.size(); i++) {
			if (plan.inputs[i].chunk_col == col) {
				return NumericCast<int>(i);
			}
		}
		plan.inputs.push_back({col, type, width});
		return NumericCast<int>(plan.inputs.size() - 1);
	};
	for (auto &expr : data.aggregates) {
		auto &aggr = expr->Cast<BoundAggregateExpression>();
		if (aggr.IsDistinct() || aggr.GetChildren().size() > 1) {
			return plan;
		}
		// FILTER (WHERE ...): a BOUND_REF to the BOOLEAN column the projection below computed.  The operator's
		// constructor renumbers that reference into its payload chunk and keeps the child chunk's column in
		// filter_indexes (physical_hash_aggregate.cpp:168-180), which is where its Sink reads it from
		int32_t filter = -1;
		if (aggr.GetFilter()) {
			auto &f = *aggr.GetFilter();
			auto entry = op.filter_indexes.find(f);
			if (f.GetExpressionClass() != ExpressionClass::BOUND_REF || f.GetReturnType().id() != LogicalTypeId::BOOLEAN ||
			    entry == op.filter_indexes.end()) {
				return plan;
			}
			filter = staged(entry->second, B200_BOOL, 1);
			plan.has_filter = true;
		}
		auto name = aggr.Function().GetName().GetIdentifierName();
		B200AggResult res {B200AggResult::DIRECT, NumericCast<int>(plan.descs.size()), 1.0, false};
		if (name == "count_star") {
			plan.descs.push_back({B200_AGG_COUNT_STAR, B200_INT64, -1, 0});
			plan.filters.push_back(filter);
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
		int input = staged(child->Cast<BoundReferenceExpression>().Index(), in_type,
		                   GetTypeIdSize(child->GetReturnType().InternalType()));
		if (plan.inputs[input].type != in_type) {
			return plan; // (a BOOLEAN filter column read as an input of another physical type cannot occur)
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
		plan.filters.resize(plan.descs.size(), filter); // (AVG_INT: its SUM and COUNT carry the same filter)
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
	// distinct (input, filter) pairs: the aggregate's states (count_star with filter f is the pair (f, f)); without
	// filters these are the distinct inputs
	vector<std::pair<int, int>> pairs;
	for (idx_t d = 0; d < plan.descs.size(); d++) {
		auto &desc = plan.descs[d];
		if (desc.func == B200_AGG_COUNT_STAR && plan.filters[d] < 0) {
			continue;
		}
		std::pair<int, int> pair(desc.func == B200_AGG_COUNT_STAR ? plan.filters[d] : desc.input, plan.filters[d]);
		if (std::find(pairs.begin(), pairs.end(), pair) == pairs.end()) {
			pairs.push_back(pair);
		}
	}
	if (plan.descs.size() > 16 || pairs.size() > 12 || key_bytes + 1 > 32) {
		return plan;
	}
	plan.eligible = true;
	return plan;
}

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
		if (plan.has_filter) {
			B200Check(b200_agg_create_filtered(state->ctx, key_types.data(), NumericCast<int>(key_types.size()),
			                                   plan.descs.data(), plan.filters.data(), NumericCast<int>(plan.descs.size()),
			                                   0, &state->agg));
		} else {
			B200Check(b200_agg_create(state->ctx, key_types.data(), NumericCast<int>(key_types.size()),
			                          plan.descs.data(), NumericCast<int>(plan.descs.size()), 0, &state->agg));
		}
		return std::move(state);
	}

	unique_ptr<LocalSinkState> GetLocalSinkState(ExecutionContext &context) const override {
		auto state = make_uniq<B200LocalSinkState>();
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
		auto &l = input.local_state.Cast<B200LocalSinkState>();
		if (!on_device) {
			OperatorSinkInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Sink(context, chunk, inner_input);
		}
		auto &g = input.global_state.Cast<B200AggGlobalState>();
		l.staging.Feed(chunk, [&](b200_batch *batch) { SinkBatch(context, g, batch); });
		return SinkResultType::NEED_MORE_INPUT;
	}

	SinkCombineResultType Combine(ExecutionContext &context, OperatorSinkCombineInput &input) const override {
		auto &l = input.local_state.Cast<B200LocalSinkState>();
		if (!on_device) {
			OperatorSinkCombineInput inner_input {*inner.sink_state, *l.inner, input.interrupt_state};
			return inner.Combine(context, inner_input);
		}
		auto &g = input.global_state.Cast<B200AggGlobalState>();
		l.staging.Drain([&](b200_batch *batch) { SinkBatch(context, g, batch); });
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
		auto state = make_uniq<B200SourceState>();
		if (!on_device) {
			state->inner = inner.GetGlobalSourceState(context);
		}
		return std::move(state);
	}
	unique_ptr<LocalSourceState> GetLocalSourceState(ExecutionContext &context, GlobalSourceState &gstate) const override {
		auto state = make_uniq<B200LocalSourceState>();
		if (!on_device) {
			state->inner = inner.GetLocalSourceState(context, *gstate.Cast<B200SourceState>().inner);
		}
		return std::move(state);
	}

	SourceResultType GetDataInternal(ExecutionContext &context, DataChunk &chunk,
	                                 OperatorSourceInput &input) const override {
		auto &src = input.global_state.Cast<B200SourceState>();
		if (!on_device) {
			OperatorSourceInput inner_input {*src.inner, *input.local_state.Cast<B200LocalSourceState>().inner,
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
