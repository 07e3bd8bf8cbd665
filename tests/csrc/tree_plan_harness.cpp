// Test-only harness of the host compiler and work planner (batch_plan.h / batch_plan.inc) for query-tree batches
// (nrtgpu_search_tree), compiled by g++ without CUDA and loaded by tests/tree_plan_harness.py. It builds a dictionary with
// the index-build rules, compiles and plans one request with its nested queries, and hands back the product's records
// (clauses, queries, nodes), item list and counters.
#include "../../nrtsearch_b200/csrc/batch_plan.h"
#include "../../nrtsearch_b200/csrc/batch_plan.inc"

#include <memory>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

#define TH_EXPORT extern "C" __attribute__((visibility("default")))

struct ThPlan {
  std::vector<int32_t> term_plane, term_gran;
  CompiledBatch cb;
  WorkPlan plan;
};

TH_EXPORT const char* th_last_error(void) { return g_last_error.c_str(); }
TH_EXPORT int th_sizeof_clause(void) { return (int)sizeof(DevClause); }
TH_EXPORT int th_sizeof_query(void) { return (int)sizeof(DevQuery); }
TH_EXPORT int th_sizeof_node(void) { return (int)sizeof(DevNode); }

// Compile and plan one request (nodes may be NULL with n_nodes 0: a flat request) on a dictionary built with the
// index-build rules; sm_count = 0 keeps the knobs' default of an H100 SXM (132). Returns the status; *out owns the result.
TH_EXPORT int th_plan(int32_t n_docs, int32_t doc_base, int32_t n_terms, const int64_t* term_off, const int32_t* term_field,
                      const int64_t* term_df, const float* term_max_x, const int64_t* field_doc_count, int32_t n_columns,
                      const uint8_t* col_multi, const int32_t* col_n_distinct, int32_t has_deletes, int32_t sm_count,
                      const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                      const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                      const nrtgpu_sort* sort, const nrtgpu_aggregation* aggs, int32_t n_aggs, ThPlan** out) {
  std::unique_ptr<ThPlan> h(new ThPlan);
  std::vector<int32_t> planes, rn; std::vector<int64_t> ro;
  plan_planes(n_docs, n_terms, term_off, h->term_plane, planes);
  plan_gran_rows(n_docs, n_terms, term_off, h->term_gran, ro, rn);
  PlanDict d;
  d.n_docs = n_docs; d.doc_base = doc_base; d.n_terms = n_terms; d.n_columns = n_columns;
  d.term_off = term_off; d.term_field = term_field; d.term_df = term_df; d.term_max_x = term_max_x;
  d.term_plane = h->term_plane.data(); d.term_gran = h->term_gran.data(); d.field_doc_count = field_doc_count;
  d.col_multi = col_multi; d.col_n_distinct = col_n_distinct; d.has_deletes = has_deletes != 0;
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags};
  r.sort = sort; r.aggs = aggs; r.n_aggs = n_aggs;
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  PlanKnobs k;
  k.sm_count = sm_count > 0 ? sm_count : 132;
  plan_work(d, k, h->cb, &h->plan);
  *out = h.release();
  return NRTGPU_OK;
}

TH_EXPORT void th_free(ThPlan* h) { delete h; }

// [n_work, n_probe_simple, n_probe_generic, parts_max, n_lists, n_slices, slice_docs, n_gran, wide, alg_postings,
//  threshold, n_clauses, tree, n_nodes]
TH_EXPORT void th_counters(const ThPlan* h, int64_t* out) {
  const WorkPlan& p = h->plan;
  const int64_t v[] = {p.n_work(), p.n_probe_simple, p.n_probe_generic, p.parts_max, p.n_lists, p.n_slices, p.slice_docs,
                       p.n_gran, h->cb.wide ? 1 : 0, h->cb.alg_postings, h->cb.threshold, (int64_t)h->cb.clauses.size(),
                       h->cb.tree ? 1 : 0, (int64_t)h->cb.nodes.size()};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

TH_EXPORT void th_items(const ThPlan* h, int32_t* work_query, int32_t* work_item) {
  std::copy(h->plan.work_query.begin(), h->plan.work_query.end(), work_query);
  std::copy(h->plan.work_item.begin(), h->plan.work_item.end(), work_item);
}

// the DevClause / DevQuery records, and for a tree batch the DevNode records and the [nq + 1] node ranges
TH_EXPORT void th_records(const ThPlan* h, void* clauses, void* queries, void* nodes, int32_t* node_begin) {
  std::memcpy(clauses, h->cb.clauses.data(), h->cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, h->cb.queries.data(), h->cb.queries.size() * sizeof(DevQuery));
  std::memcpy(nodes, h->cb.nodes.data(), h->cb.nodes.size() * sizeof(DevNode));
  std::copy(h->cb.node_begin.begin(), h->cb.node_begin.end(), node_begin);
}
