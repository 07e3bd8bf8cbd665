// Test-only harness of the host compiler (batch_plan.h / batch_plan.inc) for query trees with block joins
// (NRTGPU_NODE_NESTED), compiled by g++ without CUDA and loaded by tests/nested_plan_harness.py. It compiles one request as
// nrtgpu_search_tree_phrases does (joins and multi-phrases accepted), on an image with or without parents and with a join
// cap, plans its work, and hands back the records, the joins and the child pass's work items.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

#include <memory>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define NJ_EXPORT extern "C" __attribute__((visibility("default")))

struct NjPlan {
  std::vector<int32_t> term_plane, term_gran;
  CompiledBatch cb;
  WorkPlan wp;
};

NJ_EXPORT const char* nj_last_error(void) { return g_last_error.c_str(); }

// Compile and plan one request; n_parents < 0: an image without parents; max_join_children <= 0: the product's cap.
// Returns the status; *out owns the result.
NJ_EXPORT int nj_plan(int32_t n_docs, int32_t n_terms, const int64_t* term_off, const int32_t* term_field, const int64_t* term_df,
                      const float* term_max_x, const int64_t* field_doc_count, int64_t n_parents, int64_t max_join_children,
                      const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                      const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms,
                      const nrtgpu_query* queries, int32_t nq, int32_t top_k, NjPlan** out) {
  std::unique_ptr<NjPlan> h(new NjPlan);
  std::vector<int32_t> planes, rn; std::vector<int64_t> ro;
  plan_planes(n_docs, n_terms, term_off, h->term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, h->term_gran, ro, rn);
  static const uint8_t no_multi = 0; static const int32_t no_distinct = 0;
  PlanDict d;
  d.n_docs = n_docs; d.n_terms = n_terms;
  d.term_off = term_off; d.term_field = term_field; d.term_df = term_df; d.term_max_x = term_max_x;
  d.term_plane = h->term_plane.data(); d.term_gran = h->term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = &no_multi; d.col_n_distinct = &no_distinct;
  d.has_positions = true;
  d.has_parents = n_parents >= 0; d.n_parents = std::max<int64_t>(n_parents, 0);
  if (max_join_children > 0) d.max_join_children = max_join_children;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, 0};
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  if (n_phrases > 0) { r.phrases = phrases; r.n_phrases = n_phrases; r.phrase_terms = phrase_terms; r.n_phrase_terms = n_phrase_terms; }
  r.unions = true; r.joins = true;
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  PlanKnobs kn; kn.sm_count = 132;
  plan_work(d, kn, h->cb, &h->wp);
  *out = h.release();
  return NRTGPU_OK;
}

NJ_EXPORT void nj_free(NjPlan* h) { delete h; }

// [n_clauses, n_queries (request + child), n_nodes, n_joins, join_bound, n_work, n_join_work, n_slices]
NJ_EXPORT void nj_counters(const NjPlan* h, int64_t* out) {
  const CompiledBatch& cb = h->cb;
  const int64_t v[] = {(int64_t)cb.clauses.size(), (int64_t)cb.queries.size(), (int64_t)cb.nodes.size(), cb.n_joins(), cb.join_bound,
                       h->wp.n_work(), (int64_t)h->wp.join_query.size(), h->wp.n_slices};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// the DevClause / DevQuery / DevNode records, the [n_queries + 1] node ranges, the joins' clauses and modes, the work
// items (query per item) of the parent pass and of the child pass
NJ_EXPORT void nj_records(const NjPlan* h, void* clauses, void* queries, void* nodes, int32_t* node_begin, int32_t* join_clause,
                          uint8_t* join_mode, int32_t* work_query, int32_t* join_query) {
  const CompiledBatch& cb = h->cb;
  std::memcpy(clauses, cb.clauses.data(), cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, cb.queries.data(), cb.queries.size() * sizeof(DevQuery));
  std::memcpy(nodes, cb.nodes.data(), cb.nodes.size() * sizeof(DevNode));
  std::copy(cb.node_begin.begin(), cb.node_begin.end(), node_begin);
  std::copy(cb.join_clause.begin(), cb.join_clause.end(), join_clause);
  std::copy(cb.join_mode.begin(), cb.join_mode.end(), join_mode);
  std::copy(h->wp.work_query.begin(), h->wp.work_query.end(), work_query);
  std::copy(h->wp.join_query.begin(), h->wp.join_query.end(), join_query);
}
