// Test-only harness of the host compiler and work planner (batch_plan.h / batch_plan.inc) for the collector requests of
// nrtgpu_search_tree_aggs, compiled by g++ without CUDA and loaded by tests/window_aggs_plan_harness.py. It builds a
// dictionary with the index-build rules, compiles and plans one request -- query trees, phrases, aggregations, nested
// collectors, their sort orders and filter records -- with or without window_collectors, and hands back the product's
// counters, collector records, DevClause / DevQuery records and item list. Sort orders are opaque to the compiler, so any
// non-NULL address stands for one.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

#include <memory>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define WAH_EXPORT extern "C" __attribute__((visibility("default")))

struct WahPlan {
  std::vector<int32_t> term_plane, term_gran;
  CompiledBatch cb;
  WorkPlan plan;
};

WAH_EXPORT const char* wah_last_error(void) { return g_last_error.c_str(); }
WAH_EXPORT int wah_sizeof_clause(void) { return (int)sizeof(DevClause); }
WAH_EXPORT int wah_sizeof_query(void) { return (int)sizeof(DevQuery); }

// Compile and plan one request on a dictionary built with the index-build rules (knobs of an H100 SXM: 132 SMs); the
// request is that of nrtgpu_search_tree_aggs (threshold INT32_MAX) with window_collectors as given. Returns the status;
// *out owns the result.
WAH_EXPORT int wah_plan(int32_t n_docs, int32_t n_terms, const int64_t* term_off, const int32_t* term_field, const int64_t* term_df,
                        const float* term_max_x, const int64_t* field_doc_count, int32_t n_columns, const uint8_t* col_multi,
                        const int32_t* col_n_distinct, int32_t has_positions, const nrtgpu_clause* clauses, int32_t n_clauses,
                        const nrtgpu_node* nodes, int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                        const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries, int32_t nq,
                        int32_t top_k, const nrtgpu_sort* sort, const nrtgpu_aggregation* aggs, int32_t n_aggs,
                        const nrtgpu_nested_aggregation* nested, int32_t n_nested, const nrtgpu_nested_sort* nested_sorts,
                        const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                        const nrtgpu_query* filter_queries, int32_t n_filter_queries, int32_t window_collectors, WahPlan** out) {
  std::unique_ptr<WahPlan> h(new WahPlan);
  std::vector<int32_t> planes, rn; std::vector<int64_t> ro;
  plan_planes(n_docs, n_terms, term_off, h->term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, h->term_gran, ro, rn);
  PlanDict d;
  d.n_docs = n_docs; d.n_terms = n_terms; d.n_columns = n_columns;
  d.term_off = term_off; d.term_field = term_field; d.term_df = term_df; d.term_max_x = term_max_x;
  d.term_plane = h->term_plane.data(); d.term_gran = h->term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct; d.has_positions = has_positions != 0;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, 0};
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  if (n_phrases > 0) { r.phrases = phrases; r.n_phrases = n_phrases; r.phrase_terms = phrase_terms; r.n_phrase_terms = n_phrase_terms; }
  r.sort = sort;
  r.aggs = aggs; r.n_aggs = n_aggs;
  if (n_nested > 0) { r.nested = nested; r.n_nested = n_nested; r.nested_sorts = nested_sorts; }
  r.agg_filters = agg_filters; r.filter_clauses = filter_clauses; r.n_filter_clauses = n_filter_clauses;
  r.filter_queries = filter_queries; r.n_filter_queries = n_filter_queries;
  r.window_collectors = window_collectors != 0;
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  PlanKnobs k;
  k.sm_count = 132;
  plan_work(d, k, h->cb, &h->plan);
  *out = h.release();
  return NRTGPU_OK;
}

WAH_EXPORT void wah_free(WahPlan* h) { delete h; }

// [n_work, n_probe_simple, n_probe_generic, n_lists, n_slices, slice_docs, wide, tree, threshold, n_clauses, n_nodes, n_phrases,
//  n_aggs, n_nested, n_sorted (nested records with an order), n_filters (FILTER aggregations), agg_filter_queries]
WAH_EXPORT void wah_counters(const WahPlan* h, int64_t* out) {
  const WorkPlan& p = h->plan;
  const CompiledBatch& cb = h->cb;
  int64_t n_sorted = 0, n_filters = 0;
  for (const nrtgpu_nested_sort& s : cb.nested_sorts) n_sorted += s.orders != nullptr;
  for (const nrtgpu_aggregation& a : cb.aggs) n_filters += a.kind == NRTGPU_AGG_FILTER;
  const int64_t v[] = {p.n_work(), p.n_probe_simple, p.n_probe_generic, p.n_lists, p.n_slices, p.slice_docs, cb.wide ? 1 : 0,
                       cb.tree ? 1 : 0, cb.threshold, (int64_t)cb.clauses.size(), (int64_t)cb.nodes.size(), (int64_t)cb.phrases.size(),
                       (int64_t)cb.aggs.size(), (int64_t)cb.nested.size(), n_sorted, n_filters, cb.agg_filter_queries ? 1 : 0};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// the compiled aggregation and nested records, in request order
WAH_EXPORT void wah_collectors(const WahPlan* h, nrtgpu_aggregation* aggs, nrtgpu_nested_aggregation* nested) {
  std::copy(h->cb.aggs.begin(), h->cb.aggs.end(), aggs);
  std::copy(h->cb.nested.begin(), h->cb.nested.end(), nested);
}

// the DevClause / DevQuery records and the item list
WAH_EXPORT void wah_records(const WahPlan* h, void* clauses, void* queries, int32_t* work_query, int32_t* work_item) {
  std::memcpy(clauses, h->cb.clauses.data(), h->cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, h->cb.queries.data(), h->cb.queries.size() * sizeof(DevQuery));
  std::copy(h->plan.work_query.begin(), h->plan.work_query.end(), work_query);
  std::copy(h->plan.work_item.begin(), h->plan.work_item.end(), work_item);
}
