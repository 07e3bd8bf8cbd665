// Test-only harness of the keyword-terms checks of the host batch compiler (compile_batch in batch_plan.inc) and of
// nrtgpu_index_add_keyword_columns (check_keyword_columns), compiled by g++ without CUDA and loaded by
// tests/test_keyword_aggs_plan.py: requests compiled on a dictionary of numeric and keyword columns alone (no terms, no
// postings).
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define KPH_EXPORT extern "C" __attribute__((visibility("default")))

KPH_EXPORT const char* kph_last_error(void) { return g_last_error.c_str(); }
KPH_EXPORT int kph_sizeof_keyword_column(void) { return (int)sizeof(nrtgpu_keyword_column); }

// compile_batch of nq match-all queries with these collectors on a shard of n_docs docs, n_columns numeric columns
// (col_multi, col_n_distinct) and n_keyword keyword columns (kw_n_terms); returns the status, out_n_aggs the
// aggregations compiled
KPH_EXPORT int kph_compile(int32_t n_docs, int32_t n_columns, const uint8_t* col_multi, const int32_t* col_n_distinct, int32_t n_keyword,
                           const int32_t* kw_n_terms, int32_t nq, const nrtgpu_aggregation* aggs, int32_t n_aggs,
                           const nrtgpu_nested_aggregation* nested, int32_t n_nested, int32_t* out_n_aggs) {
  const int64_t term_off[1] = {0};
  const int64_t field_doc_count[1] = {n_docs};
  PlanDict d;
  d.n_docs = n_docs; d.n_columns = n_columns; d.term_off = term_off; d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct;
  d.n_keyword = n_keyword; d.kw_n_terms = kw_n_terms;
  std::vector<nrtgpu_clause> cl((size_t)nq);
  std::vector<nrtgpu_query> qs((size_t)nq);
  for (int q = 0; q < nq; ++q) {
    std::memset(&cl[(size_t)q], 0, sizeof(nrtgpu_clause));
    cl[(size_t)q].occur = NRTGPU_MUST; cl[(size_t)q].kind = NRTGPU_MATCH_ALL; cl[(size_t)q].boost = 1.0f;
    std::memset(&qs[(size_t)q], 0, sizeof(nrtgpu_query));
    qs[(size_t)q].clause_begin = q; qs[(size_t)q].clause_end = q + 1;
  }
  BatchRequest r{cl.data(), nq, qs.data(), nq, 10, INT32_MAX, 0};
  r.aggs = aggs; r.n_aggs = n_aggs; r.nested = nested; r.n_nested = n_nested;
  CompiledBatch cb;
  const int rc = compile_batch(d, r, &cb);
  if (!rc && out_n_aggs) *out_n_aggs = (int32_t)cb.aggs.size();
  return rc;
}

// the checks of nrtgpu_index_add_keyword_columns on an image of n_docs docs
KPH_EXPORT int kph_check_keyword_columns(int32_t n_docs, const nrtgpu_keyword_column* cols, int32_t n) {
  return check_keyword_columns(n_docs, cols, n);
}
