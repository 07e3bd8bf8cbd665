// Test-only harness of the sorted-top-hits check of the host batch compiler (compile_batch in batch_plan.inc), compiled by
// g++ without CUDA and loaded by tests/test_sorted_hits_plan.py: the request of tests/csrc/filter_plan_harness.cpp plus the
// nrtgpu_nested_sort array. Sort orders are opaque to the compiler, so any non-NULL address stands for one.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define SHP_EXPORT extern "C" __attribute__((visibility("default")))

SHP_EXPORT const char* shp_last_error(void) { return g_last_error.c_str(); }
SHP_EXPORT int shp_sizeof_nested_sort(void) { return (int)sizeof(nrtgpu_nested_sort); }

// compile_batch of nq match-all queries with these collectors on a shard of n_docs docs and n_columns columns (col_multi,
// col_n_distinct); returns the status, out_n_sorted the nested records compiled with an order
SHP_EXPORT int shp_compile(int32_t n_docs, int32_t n_columns, const uint8_t* col_multi, const int32_t* col_n_distinct, int32_t nq,
                           const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                           const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                           const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                           int32_t n_filter_queries, int32_t* out_n_sorted) {
  const int64_t term_off[1] = {0};
  const int64_t field_doc_count[1] = {n_docs};
  PlanDict d;
  d.n_docs = n_docs; d.n_columns = n_columns; d.term_off = term_off; d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct;
  std::vector<nrtgpu_clause> cl((size_t)nq);
  std::vector<nrtgpu_query> qs((size_t)nq);
  for (int q = 0; q < nq; ++q) {
    std::memset(&cl[(size_t)q], 0, sizeof(nrtgpu_clause));
    cl[(size_t)q].occur = NRTGPU_MUST; cl[(size_t)q].kind = NRTGPU_MATCH_ALL; cl[(size_t)q].boost = 1.0f;
    std::memset(&qs[(size_t)q], 0, sizeof(nrtgpu_query));
    qs[(size_t)q].clause_begin = q; qs[(size_t)q].clause_end = q + 1;
  }
  BatchRequest r{cl.data(), nq, qs.data(), nq, 10, INT32_MAX, 0};
  r.aggs = aggs; r.n_aggs = n_aggs; r.nested = nested; r.n_nested = n_nested; r.nested_sorts = nested_sorts;
  r.agg_filters = agg_filters; r.filter_clauses = filter_clauses; r.n_filter_clauses = n_filter_clauses;
  r.filter_queries = filter_queries; r.n_filter_queries = n_filter_queries;
  CompiledBatch cb;
  const int rc = compile_batch(d, r, &cb);
  if (!rc && out_n_sorted) {
    *out_n_sorted = 0;
    for (const nrtgpu_nested_sort& s : cb.nested_sorts) *out_n_sorted += s.orders != nullptr;
  }
  return rc;
}
