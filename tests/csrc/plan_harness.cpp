// Test-only harness of the host batch compiler and work planner (batch_plan.h / batch_plan.inc), compiled by g++ without
// CUDA and loaded by tests/plan_harness.py. It builds a dictionary with the index-build rules, compiles and plans one
// batch, and hands back the product's records, item list and counters.
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

PH_EXPORT const char* ph_last_error(void) { return g_last_error.c_str(); }
PH_EXPORT int ph_sizeof_clause(void) { return (int)sizeof(DevClause); }
PH_EXPORT int ph_sizeof_query(void) { return (int)sizeof(DevQuery); }

// [kT, kGran, kWarmGran, kMaxSliceGran, kWideSliceDocs, kProbeMaxTopK, kMaxTopK, warm_min_docs, slice_gran, item_postings]
PH_EXPORT void ph_constants(int64_t* out) {
  const PlanKnobs k;
  const int64_t v[] = {v3::kT, v3::kGran, v3::kWarmGran, v3::kMaxSliceGran, kWideSliceDocs, v3::kProbeMaxTopK, kMaxTopK,
                       k.warm_min_docs, k.slice_gran, k.item_postings};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// the index-build rules: tf plane and granule row of every term
PH_EXPORT void ph_index_rules(int32_t n_docs, int32_t n_terms, const int64_t* term_off, int32_t* term_plane, int32_t* term_gran) {
  std::vector<int32_t> tp, tg, planes; std::vector<int64_t> ro; std::vector<int32_t> rn;
  plan_planes(n_docs, n_terms, term_off, tp, planes);
  plan_gran_rows(n_docs, n_terms, term_off, tg, ro, rn);
  std::copy(tp.begin(), tp.end(), term_plane);
  std::copy(tg.begin(), tg.end(), term_gran);
}

PH_EXPORT void ph_bm25_cache(float k1, float b, float avgdl, float* cache) { bm25_cache(k1, b, avgdl, cache); }

// Compile and (plan != 0) plan one batch on a dictionary built with the index-build rules; sm_count = 0 keeps the
// knobs' default of an H100 SXM (132). Returns the status; *out owns the result (ph_free).
PH_EXPORT int ph_plan(int32_t n_docs, int32_t doc_base, int32_t n_terms, const int64_t* term_off, const int32_t* term_field,
                      const int64_t* term_df, const float* term_max_x, const int64_t* field_doc_count, int32_t n_columns,
                      const uint8_t* col_multi, const int32_t* col_n_distinct, int32_t has_deletes, int32_t sm_count,
                      const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                      int32_t total_hits_threshold, int32_t flags, const nrtgpu_sort* sort, const nrtgpu_aggregation* aggs,
                      int32_t n_aggs, int32_t plan, PhPlan** out) {
  std::unique_ptr<PhPlan> h(new PhPlan);
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
  int rc = compile_batch(d, r, &h->cb);
  if (rc) return rc;
  if (plan) {
    PlanKnobs k;
    k.sm_count = sm_count > 0 ? sm_count : 132;
    plan_work(d, k, h->cb, &h->plan);
  }
  *out = h.release();
  return NRTGPU_OK;
}

PH_EXPORT void ph_free(PhPlan* h) { delete h; }

// [n_work, n_probe_simple, n_probe_generic, parts_max, n_lists, n_slices, slice_docs, n_gran, wide, alg_postings,
//  threshold, n_clauses]
PH_EXPORT void ph_counters(const PhPlan* h, int64_t* out) {
  const WorkPlan& p = h->plan;
  const int64_t v[] = {p.n_work(), p.n_probe_simple, p.n_probe_generic, p.parts_max, p.n_lists, p.n_slices, p.slice_docs,
                       p.n_gran, h->cb.wide ? 1 : 0, h->cb.alg_postings, h->cb.threshold, (int64_t)h->cb.clauses.size()};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

PH_EXPORT void ph_items(const PhPlan* h, int32_t* work_query, int32_t* work_item) {
  std::copy(h->plan.work_query.begin(), h->plan.work_query.end(), work_query);
  std::copy(h->plan.work_item.begin(), h->plan.work_item.end(), work_item);
}

PH_EXPORT void ph_known_hits(const PhPlan* h, uint64_t* out) { std::copy(h->plan.known_hits.begin(), h->plan.known_hits.end(), out); }
PH_EXPORT void ph_records(const PhPlan* h, void* clauses, void* queries) {
  std::memcpy(clauses, h->cb.clauses.data(), h->cb.clauses.size() * sizeof(DevClause));
  std::memcpy(queries, h->cb.queries.data(), h->cb.queries.size() * sizeof(DevQuery));
}

// the shared decoder: [slice, part, lparts, flags, sweep slot]
PH_EXPORT void ph_decode(int32_t w, int32_t* out) {
  out[0] = v3::item_slice(w); out[1] = v3::item_part(w); out[2] = v3::item_lparts(w); out[3] = v3::item_flags(w);
  out[4] = v3::item_sweep_slot(w);
}
// [g_lo, g_hi, e_lo, e_hi, out_list] of item w in a plan (the kernel's set-up)
PH_EXPORT void ph_span(const PhPlan* h, int32_t w, int32_t* out) {
  const WorkPlan& p = h->plan;
  const int gran_per_slice = p.slice_docs / v3::kGran;
  const int fine = (gran_per_slice + p.parts_max - 1) / p.parts_max;
  const int g_count = std::min(gran_per_slice, p.n_gran - v3::item_slice(w) * gran_per_slice);
  const v3::ItemSpan s = v3::item_span(w, g_count, fine, p.parts_max, p.n_slices);
  out[0] = s.g_lo; out[1] = s.g_hi; out[2] = s.e_lo; out[3] = s.e_hi; out[4] = v3::item_out_list(w, p.parts_max, p.n_lists);
}
PH_EXPORT int64_t ph_boundary_gran(const PhPlan* h, int32_t e) {
  const WorkPlan& p = h->plan;
  return v3::boundary_gran(e, p.n_slices, p.parts_max, p.slice_docs / v3::kGran, p.n_gran);
}
