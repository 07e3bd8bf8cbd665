// Test-only harness of the host compiler and work planner (batch_plan.h / batch_plan.inc) for query-tree batches with phrase
// leaves (nrtgpu_search_tree_phrases), compiled by g++ without CUDA and loaded by tests/phrase_plan_harness.py. It builds a
// dictionary with the index-build rules, with or without positions, compiles and plans one request with its nested queries
// and its phrase table, and hands back the product's records (clauses, queries, nodes, phrase records).
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

#include <memory>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define PH_EXPORT extern "C" __attribute__((visibility("default")))

struct PhPlan {
  std::vector<int32_t> term_plane, term_gran;
  CompiledBatch cb;
  WorkPlan plan;
};

PH_EXPORT const char* pp_last_error(void) { return g_last_error.c_str(); }
PH_EXPORT int pp_sizeof_clause(void) { return (int)sizeof(DevClause); }
PH_EXPORT int pp_sizeof_query(void) { return (int)sizeof(DevQuery); }
PH_EXPORT int pp_sizeof_node(void) { return (int)sizeof(DevNode); }
PH_EXPORT int pp_sizeof_phrase(void) { return (int)sizeof(DevPhrase); }

// Compile and plan one request on a dictionary built with the index-build rules (an H100 SXM's 132 SMs); has_positions
// says whether the image holds positions. Returns the status; *out owns the result.
PH_EXPORT int pp_plan(int32_t n_docs, int32_t n_terms, const int64_t* term_off, const int32_t* term_field, const int64_t* term_df,
                      const float* term_max_x, const int64_t* field_doc_count, int32_t has_positions, int32_t n_columns,
                      const uint8_t* col_multi, const int32_t* col_n_distinct, const nrtgpu_clause* clauses, int32_t n_clauses,
                      const nrtgpu_node* nodes, int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                      const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries, int32_t nq,
                      int32_t top_k, int32_t total_hits_threshold, PhPlan** out) {
  std::unique_ptr<PhPlan> h(new PhPlan);
  std::vector<int32_t> planes, rn; std::vector<int64_t> ro;
  plan_planes(n_docs, n_terms, term_off, h->term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, h->term_gran, ro, rn);
  PlanDict d;
  d.n_docs = n_docs; d.n_terms = n_terms; d.n_columns = n_columns;
  d.term_off = term_off; d.term_field = term_field; d.term_df = term_df; d.term_max_x = term_max_x;
  d.term_plane = h->term_plane.data(); d.term_gran = h->term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct;
  d.has_positions = has_positions != 0;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, 0};
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  if (n_phrases > 0) { r.phrases = phrases; r.n_phrases = n_phrases; r.phrase_terms = phrase_terms; r.n_phrase_terms = n_phrase_terms; }
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  PlanKnobs k;
  k.sm_count = 132;
  plan_work(d, k, h->cb, &h->plan);
  *out = h.release();
  return NRTGPU_OK;
}

PH_EXPORT void pp_free(PhPlan* h) { delete h; }

// [n_clauses, nq, n_nodes, n_phrases, tree, alg_postings, n_work]
PH_EXPORT void pp_counters(const PhPlan* h, int64_t* out) {
  const int64_t v[] = {(int64_t)h->cb.clauses.size(), (int64_t)h->cb.queries.size(), (int64_t)h->cb.nodes.size(),
                       (int64_t)h->cb.phrases.size(), h->cb.tree ? 1 : 0, h->cb.alg_postings, h->plan.n_work()};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// the DevClause / DevQuery / DevNode / DevPhrase records and, for a tree batch, the [nq + 1] node and phrase ranges
PH_EXPORT void pp_records(const PhPlan* h, void* clauses, void* queries, void* nodes, int32_t* node_begin, void* phrases,
                          int32_t* phrase_begin) {
  std::memcpy(clauses, h->cb.clauses.data(), h->cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, h->cb.queries.data(), h->cb.queries.size() * sizeof(DevQuery));
  std::memcpy(nodes, h->cb.nodes.data(), h->cb.nodes.size() * sizeof(DevNode));
  std::copy(h->cb.node_begin.begin(), h->cb.node_begin.end(), node_begin);
  std::memcpy(phrases, h->cb.phrases.data(), h->cb.phrases.size() * sizeof(DevPhrase));
  std::copy(h->cb.phrase_begin.begin(), h->cb.phrase_begin.end(), phrase_begin);
}
