// Test-only harness of keyword range clauses in the host batch compiler (batch_plan.inc): the bounds -> code range rule
// (keyword_range_codes, keyword_seek_code) on a dictionary given as bytes and offsets, and the compilation of flat and tree
// batches holding NRTGPU_KEYWORD_RANGE clauses on a dictionary alone. Compiled by g++ without CUDA, loaded by
// tests/test_keyword_query_plan.py and tests/test_keyword_query_reference.py.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define KQH_EXPORT extern "C" __attribute__((visibility("default")))

KQH_EXPORT const char* kqh_last_error(void) { return g_last_error.c_str(); }

KQH_EXPORT int64_t kqh_seek(const uint8_t* bytes, const int64_t* off, int32_t n, const uint8_t* t, int32_t len) {
  return keyword_seek_code(bytes, off, n, t, len);
}

KQH_EXPORT int kqh_range(const uint8_t* bytes, const int64_t* off, int32_t n, const uint8_t* lower, int32_t lower_len,
                         const uint8_t* upper, int32_t upper_len, int32_t flags, int64_t* lo, int64_t* hi) {
  return keyword_range_codes(bytes, off, n, lower, lower_len, upper, upper_len, flags, lo, hi);
}

// compile_batch of a request on a dictionary of n_terms terms (one field, lists of the given lengths, df = length),
// n_columns single-valued numeric columns and n_keyword keyword columns (kw_n_terms); nodes may be NULL (a flat batch).
// Per query: out_dense its dense_driver, out_driver its driver_mask, out_nonterm has_nonterm | nonterm_scoring << 1.
KQH_EXPORT int kqh_compile(int32_t n_docs, int32_t n_terms, const int64_t* term_off, int32_t n_columns, int32_t n_keyword,
                           const int32_t* kw_n_terms, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_query* queries,
                           int32_t nq, const nrtgpu_node* nodes, int32_t n_nodes, int32_t top_k, int32_t* out_dense,
                           uint32_t* out_driver, int32_t* out_nonterm) {
  std::vector<int32_t> term_field((size_t)n_terms, 0), term_plane, term_gran, planes, rn;
  std::vector<int64_t> term_df((size_t)n_terms), ro;
  std::vector<float> term_max_x((size_t)n_terms, 1.0f);
  for (int32_t t = 0; t < n_terms; ++t) term_df[(size_t)t] = term_off[t + 1] - term_off[t];
  plan_planes(n_docs, n_terms, term_off, term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, term_gran, ro, rn);
  const int64_t field_doc_count[1] = {n_docs};
  std::vector<uint8_t> col_multi((size_t)std::max(n_columns, 1), 0);
  std::vector<int32_t> col_n_distinct((size_t)std::max(n_columns, 1), 10);
  PlanDict d;
  d.n_docs = n_docs; d.n_terms = n_terms; d.n_columns = n_columns;
  d.term_off = term_off; d.term_field = term_field.data(); d.term_df = term_df.data(); d.term_max_x = term_max_x.data();
  d.term_plane = term_plane.data(); d.term_gran = term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = col_multi.data(); d.col_n_distinct = col_n_distinct.data();
  d.n_keyword = n_keyword; d.kw_n_terms = kw_n_terms;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, 0};
  r.nodes = nodes; r.n_nodes = n_nodes;
  CompiledBatch cb;
  const int rc = compile_batch(d, r, &cb);
  if (rc) return rc;
  for (int q = 0; q < nq; ++q) {
    out_dense[q] = cb.queries[(size_t)q].dense_driver;
    out_driver[q] = cb.queries[(size_t)q].driver_mask;
    out_nonterm[q] = cb.queries[(size_t)q].has_nonterm | (cb.queries[(size_t)q].nonterm_scoring << 1);
  }
  return NRTGPU_OK;
}

// compile_batch of nq match-all queries with one FILTER aggregation per agg_filters record (each with a nested MIN on
// numeric column 0) on the dictionary of kqh_compile without terms
KQH_EXPORT int kqh_compile_filters(int32_t n_keyword, const int32_t* kw_n_terms, const nrtgpu_agg_filter* filters, int32_t n_filters) {
  const int64_t term_off[1] = {0};
  const int64_t field_doc_count[1] = {100};
  const uint8_t col_multi[1] = {0};
  const int32_t col_n_distinct[1] = {10};
  PlanDict d;
  d.n_docs = 100; d.n_columns = 1; d.term_off = term_off; d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct; d.n_keyword = n_keyword; d.kw_n_terms = kw_n_terms;
  nrtgpu_clause cl; std::memset(&cl, 0, sizeof(cl));
  cl.occur = NRTGPU_MUST; cl.kind = NRTGPU_MATCH_ALL; cl.boost = 1.0f;
  nrtgpu_query q; std::memset(&q, 0, sizeof(q));
  q.clause_end = 1;
  std::vector<nrtgpu_aggregation> aggs((size_t)n_filters);
  std::vector<nrtgpu_nested_aggregation> nested((size_t)n_filters);
  for (int i = 0; i < n_filters; ++i) {
    std::memset(&aggs[(size_t)i], 0, sizeof(nrtgpu_aggregation));
    aggs[(size_t)i].kind = NRTGPU_AGG_FILTER;
    std::memset(&nested[(size_t)i], 0, sizeof(nrtgpu_nested_aggregation));
    nested[(size_t)i].parent = i; nested[(size_t)i].kind = NRTGPU_AGG_MIN;
  }
  BatchRequest r{&cl, 1, &q, 1, 10, INT32_MAX, 0};
  r.aggs = aggs.data(); r.n_aggs = n_filters; r.nested = nested.data(); r.n_nested = n_filters; r.agg_filters = filters;
  CompiledBatch cb;
  return compile_batch(d, r, &cb);
}
