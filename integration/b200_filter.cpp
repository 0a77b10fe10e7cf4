// Reference-side binding of the filter (host C++, see INTEGRATION.md).
//
// B200BatchedFilter replaces PhysicalFilter::ExecuteInternal (src/execution/operator/filter/physical_filter.cpp:53-64)
// when a device is present and the whole predicate translates.  It buffers input chunks (deep copies + the predicate's
// columns in the worker's pinned staging ring) until B200_FILTER_BATCH rows (default 128 K) are there, evaluates the
// predicate with ONE b200_filter_project call (out_sel = the surviving row ids, in input order) and emits the
// survivors as slices of the buffered chunks (HAVE_MORE_OUTPUT, then FinalExecute for the tail) - the same shape as
// the batched probe of B200HashJoin.  A CachingPhysicalOperator cannot batch (Execute / FinalExecute are final there),
// hence a PhysicalOperator of its own.
//
// What it shows: (1) how a bound expression tree maps onto b200_expr_node, (2) the error convention (status code ->
// duckdb::Exception), (3) that the output is produced exactly like the stock operator (chunk.Slice(input, sel, n)
// with the selection the kernel returned, or chunk.Reference(input)).
//
// B200Filter is PhysicalFilter under the binding's name: it is planned without a device and for predicates that do
// not translate, and every chunk takes the base class (the stock CPU path).
#include "b200_binding.hpp"

#include "duckdb/execution/expression_executor.hpp"
#include "duckdb/execution/operator/filter/physical_filter.hpp"
#include "duckdb/execution/physical_operator.hpp"
#include "duckdb/planner/expression/bound_comparison_expression.hpp"
#include "duckdb/planner/expression/bound_conjunction_expression.hpp"
#include "duckdb/planner/expression/bound_constant_expression.hpp"
#include "duckdb/planner/expression/bound_function_expression.hpp"
#include "duckdb/planner/expression/bound_reference_expression.hpp"

namespace duckdb {

//! Bound expression tree -> b200_expr_node program (children before parents).  Returns the root or -1.
static int TranslateExpression(const Expression &expr, vector<b200_expr_node> &prog) {
	b200_expr_node node;
	memset(&node, 0, sizeof(node));
	node.left = node.right = -1;
	int32_t type;
	if (!B200Type(expr.GetReturnType().InternalType(), type)) {
		return -1;
	}
	node.type = type;
	switch (expr.GetExpressionClass()) {
	case ExpressionClass::BOUND_REF: {
		node.op = B200_EXPR_COLREF;
		node.col = NumericCast<int32_t>(expr.Cast<BoundReferenceExpression>().Index());
		break;
	}
	case ExpressionClass::BOUND_CONSTANT: {
		auto &value = expr.Cast<BoundConstantExpression>().GetValue();
		node.op = B200_EXPR_CONST;
		node.is_null = value.IsNull();
		if (!value.IsNull()) {
			// the PHYSICAL value (DATE = int32 days, DECIMAL = scaled integer), sign- / zero-extended
			switch (expr.GetReturnType().InternalType()) {
			case PhysicalType::DOUBLE:
				node.value.d = value.GetValueUnsafe<double>();
				break;
			case PhysicalType::FLOAT:
				node.value.f = value.GetValueUnsafe<float>();
				break;
			case PhysicalType::BOOL:
				node.value.u = value.GetValueUnsafe<bool>() ? 1 : 0;
				break;
			case PhysicalType::UINT8:
				node.value.u = value.GetValueUnsafe<uint8_t>();
				break;
			case PhysicalType::UINT16:
				node.value.u = value.GetValueUnsafe<uint16_t>();
				break;
			case PhysicalType::UINT32:
				node.value.u = value.GetValueUnsafe<uint32_t>();
				break;
			case PhysicalType::UINT64:
				node.value.u = value.GetValueUnsafe<uint64_t>();
				break;
			case PhysicalType::INT8:
				node.value.i = value.GetValueUnsafe<int8_t>();
				break;
			case PhysicalType::INT16:
				node.value.i = value.GetValueUnsafe<int16_t>();
				break;
			case PhysicalType::INT32:
				node.value.i = value.GetValueUnsafe<int32_t>();
				break;
			default:
				node.value.i = value.GetValueUnsafe<int64_t>();
				break;
			}
		}
		break;
	}
	case ExpressionClass::BOUND_CONJUNCTION: {
		auto &conj = expr.Cast<BoundConjunctionExpression>();
		node.op = expr.GetExpressionType() == ExpressionType::CONJUNCTION_AND ? B200_EXPR_AND : B200_EXPR_OR;
		int acc = -1;
		for (auto &child : conj.GetChildren()) {
			int c = TranslateExpression(*child, prog);
			if (c < 0) {
				return -1;
			}
			if (acc < 0) {
				acc = c;
				continue;
			}
			b200_expr_node pair = node;
			pair.left = acc;
			pair.right = c;
			prog.push_back(pair);
			acc = NumericCast<int>(prog.size() - 1);
		}
		return acc;
	}
	case ExpressionClass::BOUND_FUNCTION: {
		if (!BoundComparisonExpression::IsComparison(expr)) {
			return -1; // arbitrary scalar functions stay on the host
		}
		auto &cmp = expr.Cast<BoundFunctionExpression>();
		node.op = static_cast<int32_t>(expr.GetExpressionType()); // COMPARE_* values are the b200 opcodes
		node.left = TranslateExpression(BoundComparisonExpression::Left(cmp), prog);
		node.right = TranslateExpression(BoundComparisonExpression::Right(cmp), prog);
		if (node.left < 0 || node.right < 0) {
			return -1;
		}
		break;
	}
	default:
		return -1;
	}
	prog.push_back(node);
	return NumericCast<int>(prog.size() - 1);
}


static idx_t B200FilterBatchRows() {
	// below one chunk (0 included) a batch is one chunk
	const char *env = getenv("B200_FILTER_BATCH");
	idx_t rows = env ? idx_t(atoll(env)) : idx_t(128) * 1024;
	return rows < STANDARD_VECTOR_SIZE ? STANDARD_VECTOR_SIZE : rows;
}

//! The predicate as a kernel program over the staged columns; eligible only when every node translates
struct B200FilterProgram {
	bool eligible = false;
	vector<b200_expr_node> nodes;
	int root = -1;
	vector<B200Column> columns; // input-chunk columns the program reads, in staging order
};

//! The kernel's expression program is bounded (B200_MAX_EXPR_NODES): a predicate that does not fit stays on the stock
//! path instead of failing at run time.  Only the columns the predicate references are staged (pass-through columns
//! of any type - VARCHAR, HUGEINT, nested - never leave the host: the output is a slice of the input).
static B200FilterProgram AnalyseFilter(const Expression &expression, const vector<LogicalType> &input_types) {
	B200FilterProgram plan;
	plan.root = TranslateExpression(expression, plan.nodes);
	if (plan.root < 0 || plan.nodes.size() > B200_MAX_EXPR_NODES) {
		return plan;
	}
	for (auto &node : plan.nodes) {
		if (node.op != B200_EXPR_COLREF) {
			continue;
		}
		idx_t chunk_col = idx_t(node.col);
		if (chunk_col >= input_types.size()) {
			return plan;
		}
		idx_t pos = 0;
		for (; pos < plan.columns.size() && plan.columns[pos].chunk_col != chunk_col; pos++) {
		}
		if (pos == plan.columns.size()) {
			int32_t type;
			auto physical = input_types[chunk_col].InternalType();
			if (!B200Type(physical, type)) {
				return plan;
			}
			plan.columns.push_back({chunk_col, type, GetTypeIdSize(physical)});
		}
		node.col = NumericCast<int32_t>(pos);
	}
	plan.eligible = !plan.columns.empty();
	return plan;
}

//! Drop-in for PhysicalFilter: same constructor, same types, same output contract, every chunk on the stock path
class B200Filter : public PhysicalFilter {
public:
	using PhysicalFilter::PhysicalFilter;

	string GetName() const override {
		return "B200_FILTER(host)";
	}

	//! EXPLAIN shows which path the operator takes
	InsertionOrderPreservingMap<string> ParamsToString() const override {
		auto result = PhysicalFilter::ParamsToString();
		result["Operator"] = GetName();
		return result;
	}
};

class B200BatchedFilterState : public B200BatchState {
public:
	B200BatchedFilterState(ExecutionContext &context, const Expression &expr) : fallback(context.client, expr) {
	}
	~B200BatchedFilterState() override {
		if (report) {
			B200TimingReport("filter (one worker's state; phases are summed over all workers since the last report)");
		}
	}
	vector<uint32_t> row_ids;               // surviving batch rows, ascending
	idx_t survivors = 0;
	ExpressionExecutor fallback;            // stock path for a batch the kernel refuses (B200_ERR_INVALID)
	bool report = true;
};

class B200BatchedFilter : public PhysicalOperator {
public:
	B200BatchedFilter(PhysicalPlan &physical_plan, vector<LogicalType> types, unique_ptr<Expression> expression_p,
	                  B200FilterProgram program_p, idx_t estimated_cardinality)
	    : PhysicalOperator(physical_plan, PhysicalOperatorType::EXTENSION, std::move(types), estimated_cardinality),
	      expression(std::move(expression_p)), program(std::move(program_p)), batch_rows(B200FilterBatchRows()) {
	}

	unique_ptr<Expression> expression;
	B200FilterProgram program;
	idx_t batch_rows;

	string GetName() const override {
		return "B200_FILTER";
	}
	InsertionOrderPreservingMap<string> ParamsToString() const override {
		InsertionOrderPreservingMap<string> result;
		result["Operator"] = "B200_FILTER (batched, " + to_string(batch_rows) + " rows per kernel call)";
		result["Expression"] = expression->ToString();
		return result;
	}
	bool ParallelOperator() const override {
		return true;
	}
	bool RequiresFinalExecute() const override {
		return true; // the last, partial batch is evaluated at the end
	}

	unique_ptr<OperatorState> GetOperatorState(ExecutionContext &context) const override {
		auto state = make_uniq<B200BatchedFilterState>(context, *expression);
		state->staging.Init(0, program.columns, batch_rows + STANDARD_VECTOR_SIZE);
		return std::move(state);
	}

	//! ONE kernel call for everything buffered; row_ids = the survivors in input order
	void FilterBatch(B200BatchedFilterState &state, b200_batch *batch) const {
		idx_t n = state.buffered_rows;
		state.survivors = 0;
		state.ReserveSel(n, batch);
		uint64_t count = 0;
		B200Timer timer(B200_T_KERNEL_CALL);
		int rc = b200_filter_project(state.staging.ctx, batch, program.nodes.data(), NumericCast<int>(program.nodes.size()),
		                             program.root, nullptr, 0, nullptr, state.sel_dev, nullptr, &count);
		b200_batch_free(batch);
		state.row_ids.resize(n + 1);
		if (rc == B200_ERR_INVALID) {
			// a shape the kernel does not take: the stock executor selects chunk by chunk
			SelectionVector sel(STANDARD_VECTOR_SIZE);
			idx_t out = 0;
			for (idx_t c = 0; c < state.buffered.size(); c++) {
				idx_t k = state.fallback.SelectExpression(*state.buffered[c], sel);
				for (idx_t i = 0; i < k; i++) {
					state.row_ids[out++] = NumericCast<uint32_t>(state.chunk_start[c] + sel.get_index(i));
				}
			}
			state.survivors = out;
			return;
		}
		B200Check(rc);
		if (count > 0 &&
		    cudaMemcpy(state.row_ids.data(), state.sel_dev, count * sizeof(uint32_t), cudaMemcpyDeviceToHost) != cudaSuccess) {
			throw IOException("b200: D2H of the selection vector failed");
		}
		state.survivors = count;
	}

	//! emit the survivors of the next buffered chunk that has any; false when the batch is drained
	bool EmitNext(B200BatchedFilterState &state, DataChunk &chunk) const {
		B200Timer timer(B200_T_EMIT);
		while (state.emit_chunk < state.buffered.size()) {
			idx_t c = state.emit_chunk++;
			auto &src = *state.buffered[c];
			idx_t begin = state.chunk_start[c], end = begin + src.size();
			idx_t first = state.emit_pos;
			while (state.emit_pos < state.survivors && state.row_ids[state.emit_pos] < end) {
				state.emit_pos++;
			}
			idx_t count = state.emit_pos - first;
			if (count == 0) {
				continue;
			}
			if (count == src.size()) {
				chunk.Reference(src); // nothing was filtered (physical_filter.cpp:57-59)
			} else {
				SelectionVector sel(STANDARD_VECTOR_SIZE);
				for (idx_t i = 0; i < count; i++) {
					sel.set_index(i, state.row_ids[first + i] - begin);
				}
				chunk.Slice(src, sel, count); // dictionary vectors over the buffered chunk, zero copy (:60-61)
			}
			return true;
		}
		return false;
	}

	OperatorResultType Execute(ExecutionContext &context, DataChunk &input, DataChunk &chunk, GlobalOperatorState &gstate,
	                           OperatorState &state_p) const override {
		auto &state = state_p.Cast<B200BatchedFilterState>();
		return state.Execute(
		    context, input, chunk, batch_rows, [&](b200_batch *batch) { FilterBatch(state, batch); },
		    [&](DataChunk &out) { return EmitNext(state, out); });
	}

	OperatorFinalizeResultType FinalExecute(ExecutionContext &context, DataChunk &chunk, GlobalOperatorState &gstate,
	                                        OperatorState &state_p) const override {
		auto &state = state_p.Cast<B200BatchedFilterState>();
		return state.FinalExecute(
		    context, chunk, [&](b200_batch *batch) { FilterBatch(state, batch); },
		    [&](DataChunk &out) { return EmitNext(state, out); });
	}
};

//! the select list of a LogicalFilter as ONE expression (PhysicalFilter's constructor, physical_filter.cpp:10-21)
static unique_ptr<Expression> ConjunctionOf(vector<unique_ptr<Expression>> select_list) {
	if (select_list.size() == 1) {
		return std::move(select_list[0]);
	}
	auto conjunction = make_uniq<BoundConjunctionExpression>(ExpressionType::CONJUNCTION_AND);
	for (auto &expr : select_list) {
		conjunction->GetChildrenMutable().push_back(std::move(expr));
	}
	return std::move(conjunction);
}

} // namespace duckdb
