// Plan insertion WITHOUT touching DuckDB's sources (INTEGRATION.md "Option A"):
//   OptimizerExtension (src/include/duckdb/optimizer/optimizer_extension.hpp:35-53, run after the built-in passes,
//   src/optimizer/optimizer.cpp:539) replaces LogicalFilter nodes by a LogicalExtensionOperator whose CreatePlan
//   (src/execution/physical_plan_generator.cpp:205-208) makes a B200Filter.
// Built by integration/build.sh against the reference headers into integration/_build/libb200_duckdb.so, which
// links libduckdb_ref.so (the unmodified reference) and libduckdb_b200.so (the kernels).  tests/test_integration.py
// registers it on a database opened through DuckDB's C API and runs BASELINE config 1 through it.
#include "b200_filter.cpp"
#include "b200_aggregate.cpp"
#include "b200_join.cpp"

#include "duckdb/execution/physical_plan_generator.hpp"
#include "duckdb/execution/operator/projection/physical_projection.hpp"
#include "duckdb/main/capi/capi_internal.hpp"
#include "duckdb/main/config.hpp"
#include "duckdb/main/database.hpp"
#include "duckdb/optimizer/optimizer_extension.hpp"
#include "duckdb/planner/operator/logical_extension_operator.hpp"
#include "duckdb/planner/operator/logical_filter.hpp"
#include "duckdb/planner/operator/logical_aggregate.hpp"
#include "duckdb/planner/operator/logical_comparison_join.hpp"
#include "duckdb/planner/operator/logical_get.hpp"
#include "duckdb/planner/expression/bound_columnref_expression.hpp"
#include "duckdb/planner/expression_iterator.hpp"
#include "duckdb/planner/filter/expression_filter.hpp"

namespace duckdb {

struct LogicalB200Filter : public LogicalExtensionOperator {
	explicit LogicalB200Filter(LogicalFilter &filter) : LogicalExtensionOperator(std::move(filter.expressions)) {
		children = std::move(filter.children);
		projection_map = std::move(filter.projection_map);
		estimated_cardinality = filter.estimated_cardinality;
		has_estimated_cardinality = filter.has_estimated_cardinality;
	}

	//! like LogicalFilter: the child's columns, optionally narrowed by a projection map
	vector<ProjectionIndex> projection_map;

	vector<ColumnBinding> GetColumnBindings() override {
		return MapBindings(children[0]->GetColumnBindings(), projection_map);
	}

	PhysicalOperator &CreatePlan(ClientContext &context, PhysicalPlanGenerator &planner) override {
		if (getenv("B200_DEBUG")) {
			fprintf(stderr, "[b200] LogicalB200Filter::CreatePlan\n");
		}
		auto &child = planner.CreatePlan(*children[0]);
		// with a device: the streaming operator (one kernel call per B200_FILTER_BATCH buffered rows) when the whole
		// predicate translates; B200Filter (PhysicalFilter run by the stock executor) otherwise and on the CPU box
		// ("plumbing, no GPU")
		auto predicate = ConjunctionOf(std::move(expressions));
		optional_ptr<PhysicalOperator> made;
		if (b200_device_count() > 0) {
			auto program = AnalyseFilter(*predicate, child.GetTypes());
			if (program.eligible) {
				made = planner.Make<B200BatchedFilter>(child.GetTypes(), std::move(predicate), std::move(program),
				                                        estimated_cardinality);
			}
		}
		if (!made) {
			vector<unique_ptr<Expression>> select_list;
			select_list.push_back(std::move(predicate));
			made = planner.Make<B200Filter>(child.GetTypes(), std::move(select_list), estimated_cardinality);
		}
		auto &filter = *made;
		filter.children.push_back(child);
		if (projection_map.empty()) {
			return filter;
		}
		// same as PhysicalPlanGenerator::CreatePlan(LogicalFilter&) (plan_filter.cpp:22-31): a projection drops
		// the columns that were only needed by the predicate
		vector<unique_ptr<Expression>> select_list;
		for (idx_t i = 0; i < projection_map.size(); i++) {
			select_list.push_back(make_uniq<BoundReferenceExpression>(types[i], projection_map[i]));
		}
		auto &proj = planner.Make<PhysicalProjection>(types, std::move(select_list), estimated_cardinality);
		proj.children.push_back(filter);
		return proj;
	}

	string GetExtensionName() const override {
		return "b200";
	}
	string GetName() const override {
		return "B200_FILTER";
	}

protected:
	void ResolveTypes() override {
		types = MapTypes(children[0]->types, projection_map);
	}
};

//! Pass-through wrapper around a LogicalAggregate: same bindings and types; CreatePlan lets the reference's planner
//! build its physical aggregate and, when that is an eligible PhysicalHashAggregate, decorates it
struct LogicalB200Aggregate : public LogicalExtensionOperator {
	explicit LogicalB200Aggregate(unique_ptr<LogicalOperator> aggregate) {
		estimated_cardinality = aggregate->estimated_cardinality;
		has_estimated_cardinality = aggregate->has_estimated_cardinality;
		children.push_back(std::move(aggregate));
	}

	vector<ColumnBinding> GetColumnBindings() override {
		return children[0]->GetColumnBindings();
	}

	PhysicalOperator &CreatePlan(ClientContext &context, PhysicalPlanGenerator &planner) override {
		auto &stock = planner.CreatePlan(*children[0]);
		if (stock.type != PhysicalOperatorType::HASH_GROUP_BY) {
			return stock; // perfect-hash / partitioned / ungrouped aggregates stay as planned
		}
		auto &hash_aggregate = stock.Cast<PhysicalHashAggregate>();
		auto plan = AnalyseAggregate(hash_aggregate);
		if (getenv("B200_DEBUG")) {
			fprintf(stderr, "[b200] hash aggregate: eligible=%d\n", (int)plan.eligible);
		}
		if (!plan.eligible) {
			return stock;
		}
		return planner.Make<B200HashAggregate>(hash_aggregate, std::move(plan));
	}

	string GetExtensionName() const override {
		return "b200";
	}
	string GetName() const override {
		return "B200_AGGREGATE";
	}

protected:
	void ResolveTypes() override {
		types = children[0]->types;
	}
};

//! Pass-through wrapper around a LogicalComparisonJoin: decorates the planned PhysicalHashJoin when it is eligible
struct LogicalB200Join : public LogicalExtensionOperator {
	explicit LogicalB200Join(unique_ptr<LogicalOperator> join) {
		estimated_cardinality = join->estimated_cardinality;
		has_estimated_cardinality = join->has_estimated_cardinality;
		children.push_back(std::move(join));
	}

	vector<ColumnBinding> GetColumnBindings() override {
		return children[0]->GetColumnBindings();
	}

	PhysicalOperator &CreatePlan(ClientContext &context, PhysicalPlanGenerator &planner) override {
		auto &stock = planner.CreatePlan(*children[0]);
		if (stock.type != PhysicalOperatorType::HASH_JOIN) {
			return stock; // nested-loop / merge / IE joins stay as planned
		}
		auto &hash_join = stock.Cast<PhysicalHashJoin>();
		auto plan = AnalyseJoin(hash_join);
		if (getenv("B200_DEBUG")) {
			fprintf(stderr, "[b200] hash join: eligible=%d\n", (int)plan.eligible);
		}
		if (!plan.eligible) {
			return stock;
		}
		return planner.Make<B200HashJoin>(hash_join, std::move(plan));
	}

	string GetExtensionName() const override {
		return "b200";
	}
	string GetName() const override {
		return "B200_JOIN";
	}

protected:
	void ResolveTypes() override {
		types = children[0]->types;
	}
};

//! true when the predicate is built only from comparisons / conjunctions / NULL tests over the column and
//! constants: the internal table-filter functions (dynamic join filters, bloom filters, optional wrappers) stay in
//! the scan, which owns their runtime state
static bool PlainPredicate(const Expression &expr) {
	switch (expr.GetExpressionClass()) {
	case ExpressionClass::BOUND_CONJUNCTION:
	case ExpressionClass::BOUND_CONSTANT:
	case ExpressionClass::BOUND_REF:
	case ExpressionClass::BOUND_OPERATOR:
		break;
	case ExpressionClass::BOUND_FUNCTION:
		if (!BoundComparisonExpression::IsComparison(expr)) {
			return false; // dynamic_filter(), bloom filters, optional wrappers, casts ...
		}
		break;
	default:
		return false;
	}
	bool plain = true;
	ExpressionIterator::EnumerateChildren(expr, [&](const Expression &child) { plain = plain && PlainPredicate(child); });
	return plain;
}

//! Scan-side filter binding (SURVEY.md section 8, row a12).  The stock optimizer pushes `col CMP const` predicates
//! into the table scan (LogicalGet::table_filters, evaluated by ColumnSegment::FilterSelection,
//! src/storage/table/column_segment.cpp:502-509), where no operator of ours would ever see them.  This rewrite is the
//! inverse of the reference's own fallback for scans without filter pushdown (plan_get.cpp:95-150): every plain
//! single-column table filter becomes an expression over the scan's column binding in a LogicalFilter above the scan
//! (TableFilter::ToExpression), the scan outputs the predicate's column again, and the filter's projection map
//! restores the scan's previous output columns - so parents keep their bindings and ReplaceFilters below turns the
//! new node into a B200Filter.  Dynamic / optional / multi-column filters stay where they are.
static void PullUpScanFilters(unique_ptr<LogicalOperator> &op) {
	auto &get = op->Cast<LogicalGet>();
	if (!get.table_filters.HasFilters() || get.children.size() != 0) {
		return;
	}
	auto &column_ids = get.GetColumnIds();
	vector<ProjectionIndex> pulled;
	vector<unique_ptr<Expression>> predicates;
	for (auto &entry : get.table_filters) {
		auto &table_filter = entry.Filter();
		if (table_filter.filter_type != TableFilterType::EXPRESSION_FILTER) {
			continue;
		}
		auto &filter = table_filter.Cast<ExpressionFilter>();
		auto scan_column = entry.GetIndex();
		if (!filter.column_indexes.empty() || !filter.expr || !PlainPredicate(*filter.expr) ||
		    scan_column.GetIndex() >= column_ids.size() || column_ids[scan_column.GetIndex()].IsVirtualColumn()) {
			continue;
		}
		auto table_column = column_ids[scan_column.GetIndex()].GetPrimaryIndex();
		if (table_column >= get.returned_types.size()) {
			continue;
		}
		BoundColumnRefExpression column(get.returned_types[table_column],
		                                ColumnBinding(get.table_index, ProjectionIndex(scan_column.GetIndex())));
		predicates.push_back(filter.ToExpression(column));
		pulled.push_back(scan_column);
	}
	if (predicates.empty()) {
		return;
	}
	for (auto &scan_column : pulled) {
		get.table_filters.RemoveFilterByColumnIndex(scan_column);
	}
	auto filter = make_uniq<LogicalFilter>();
	filter->expressions = std::move(predicates);
	if (!get.projection_ids.empty()) {
		// the scan emitted column_ids[projection_ids[i]]; it now emits every column_ids entry (bindings are
		// (table_index, position in column_ids) either way) and the filter narrows back to the old output
		filter->projection_map = get.projection_ids;
		get.projection_ids.clear();
	}
	if (get.has_estimated_cardinality) {
		filter->SetEstimatedCardinality(get.estimated_cardinality);
	}
	if (getenv("B200_DEBUG")) {
		fprintf(stderr, "[b200] pulled %zu table filter(s) out of the scan of table index %llu\n", pulled.size(),
		        (unsigned long long)get.table_index.index);
	}
	filter->children.push_back(std::move(op));
	op = std::move(filter);
}

static void ReplaceFilters(unique_ptr<LogicalOperator> &op) {
	for (auto &child : op->children) {
		ReplaceFilters(child);
	}
	// opt-in: a predicate the scan would evaluate on the host for free (zonemaps included) only belongs on the device
	// when the rows are going there anyway; per 2048-row chunk the offload is PCIe-latency-bound (bench.py e2e_duckdb)
	if (op->type == LogicalOperatorType::LOGICAL_GET && getenv("B200_SCAN_FILTERS") && !getenv("B200_NO_FILTER")) {
		PullUpScanFilters(op);
	}
	if (op->type == LogicalOperatorType::LOGICAL_COMPARISON_JOIN && !getenv("B200_NO_JOIN")) {
		op = make_uniq<LogicalB200Join>(std::move(op));
		return;
	}
	if (op->type == LogicalOperatorType::LOGICAL_AGGREGATE_AND_GROUP_BY && !getenv("B200_NO_AGGREGATE")) {
		auto &aggregate = op->Cast<LogicalAggregate>();
		if (!aggregate.groups.empty() && aggregate.grouping_sets.size() <= 1) {
			op = make_uniq<LogicalB200Aggregate>(std::move(op));
		}
		return;
	}
	if (op->type == LogicalOperatorType::LOGICAL_FILTER && !getenv("B200_NO_FILTER")) {
		auto &filter = op->Cast<LogicalFilter>();
		if (getenv("B200_DEBUG")) {
			fprintf(stderr, "[b200] filter node: projmap=%d exprs=%zu children=%zu\n", (int)filter.HasProjectionMap(),
			        filter.expressions.size(), filter.children.size());
		}
		if (!filter.expressions.empty() && filter.children.size() == 1) {
			op = make_uniq<LogicalB200Filter>(filter);
		}
	}
}

static void B200Optimize(OptimizerExtensionInput &input, unique_ptr<LogicalOperator> &plan) {
	if (getenv("B200_DEBUG")) {
		fprintf(stderr, "[b200] optimizer hook: %s\n", plan->ToString().c_str());
	}
	if (getenv("B200_DISABLE")) {
		return; // stock plans (bench.py times both in the same connection)
	}
	ReplaceFilters(plan);
}

} // namespace duckdb

//! Register the optimizer hook on a database opened with duckdb_open (C API handle).
extern "C" __attribute__((visibility("default"))) int b200_duckdb_register(duckdb_database db) {
	if (!db) {
		return -1;
	}
	auto wrapper = reinterpret_cast<duckdb::DatabaseWrapper *>(db);
	auto &config = duckdb::DBConfig::GetConfig(*wrapper->database->instance);
	duckdb::OptimizerExtension ext;
	ext.optimize_function = duckdb::B200Optimize;
	duckdb::OptimizerExtension::Register(config, ext);
	return 0;
}
