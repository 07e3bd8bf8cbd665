// Test-only harness of the host compiler (batch_plan.h / batch_plan.inc) for query trees with multi-phrase leaves
// (NRTGPU_MULTI_PHRASE, nrtgpu_search_tree_phrases), compiled by g++ without CUDA and loaded by
// tests/multi_phrase_plan_harness.py. It compiles one request as tests/csrc/phrase_plan_harness.cpp does, with the
// request accepting multi-phrases, the image's per-term position counts and a union postings cap, and hands back the
// product's records and the batch's distinct unions.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

#include <memory>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define MP_EXPORT extern "C" __attribute__((visibility("default")))

struct MpPlan {
  std::vector<int32_t> term_plane, term_gran;
  CompiledBatch cb;
};

MP_EXPORT const char* mp_last_error(void) { return g_last_error.c_str(); }

// Compile one request; term_pos: [n_terms + 1] first position of each term (NULL: an image without positions);
// max_union_postings <= 0: the product's cap. Returns the status; *out owns the result.
MP_EXPORT int mp_plan(int32_t n_docs, int32_t n_terms, const int64_t* term_off, const int32_t* term_field, const int64_t* term_df,
                      const float* term_max_x, const int64_t* field_doc_count, const int64_t* term_pos, int64_t max_union_postings,
                      const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                      const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms,
                      const nrtgpu_query* queries, int32_t nq, int32_t top_k, MpPlan** out) {
  std::unique_ptr<MpPlan> h(new MpPlan);
  std::vector<int32_t> planes, rn; std::vector<int64_t> ro;
  plan_planes(n_docs, n_terms, term_off, h->term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, h->term_gran, ro, rn);
  static const uint8_t no_multi = 0; static const int32_t no_distinct = 0;
  PlanDict d;
  d.n_docs = n_docs; d.n_terms = n_terms;
  d.term_off = term_off; d.term_field = term_field; d.term_df = term_df; d.term_max_x = term_max_x;
  d.term_plane = h->term_plane.data(); d.term_gran = h->term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = &no_multi; d.col_n_distinct = &no_distinct;
  d.has_positions = term_pos != nullptr; d.term_pos = term_pos;
  if (max_union_postings > 0) d.max_union_postings = max_union_postings;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, 0};
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  if (n_phrases > 0) { r.phrases = phrases; r.n_phrases = n_phrases; r.phrase_terms = phrase_terms; r.n_phrase_terms = n_phrase_terms; }
  r.unions = true;
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  *out = h.release();
  return NRTGPU_OK;
}

MP_EXPORT void mp_free(MpPlan* h) { delete h; }

// [n_clauses, nq, n_nodes, n_phrases, n_unions, n_union_terms, n_union_clauses, union_postings, union_positions]
MP_EXPORT void mp_counters(const MpPlan* h, int64_t* out) {
  const CompiledBatch& cb = h->cb;
  const int64_t v[] = {(int64_t)cb.clauses.size(), (int64_t)cb.queries.size(), (int64_t)cb.nodes.size(), (int64_t)cb.phrases.size(),
                       cb.n_unions(), (int64_t)cb.union_term.size(), (int64_t)cb.union_clause.size(), cb.union_postings,
                       cb.union_positions};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// the DevClause / DevQuery / DevPhrase records, the [nq + 1] phrase ranges, and the unions: [n_unions + 1] ranges of their
// terms and weights, their modes and the union clauses
MP_EXPORT void mp_records(const MpPlan* h, void* clauses, void* queries, void* phrases, int32_t* phrase_begin, int32_t* union_begin,
                          int32_t* union_term, float* union_weight, uint8_t* union_mode, int32_t* union_clause) {
  const CompiledBatch& cb = h->cb;
  std::memcpy(clauses, cb.clauses.data(), cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, cb.queries.data(), cb.queries.size() * sizeof(DevQuery));
  std::memcpy(phrases, cb.phrases.data(), cb.phrases.size() * sizeof(DevPhrase));
  std::copy(cb.phrase_begin.begin(), cb.phrase_begin.end(), phrase_begin);
  std::copy(cb.union_begin.begin(), cb.union_begin.end(), union_begin);
  std::copy(cb.union_term.begin(), cb.union_term.end(), union_term);
  std::copy(cb.union_weight.begin(), cb.union_weight.end(), union_weight);
  std::copy(cb.union_scored.begin(), cb.union_scored.end(), union_mode);
  std::copy(cb.union_clause.begin(), cb.union_clause.end(), union_clause);
}
