// nrtgpu.cu -- C ABI (include/nrtgpu.h) of the H100 query-execution engine: context, HBM index image,
// batch compilation, kernel launches. No CPU fallback: every entry point needs a CUDA device.
#include "../../include/nrtgpu.h"
#include "bool_kernel.cuh"
#include "join_kernel.cuh"
#include "probe_kernel.cuh"
#include "sort_kernel.cuh"
#include "collect_kernel.cuh"
#include "knn_kernel.cuh"
#include "knn_filter_kernel.cuh"
#include "hybrid_kernel.cuh"

#include <thrust/unique.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <thread>
#include <unordered_map>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>
#include <optional>
#include <vector>

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
#include "batch_plan.inc"
using namespace nrtgpu;

// index-time impacts: max over a term's postings of x = tf * cache[norm] (what Lucene keeps as competitive (freq, norm)
// pairs in its skip data); the BM25 score is monotone in x, so score(weight, max x) bounds the whole list.
// One warp per term (lists of thousands of postings take a whole CTA's worth of iterations, the millions of tiny lists one
// each): no per-posting dictionary search, no atomics.
__global__ void term_max_x_kernel(const int64_t* __restrict__ term_off, int n_terms, const int32_t* __restrict__ term_field,
                                  const int32_t* __restrict__ docs, const uint8_t* __restrict__ f8,
                                  const int64_t* __restrict__ exc_pos, const int32_t* __restrict__ exc_freq, int n_exc,
                                  const uint8_t* const* __restrict__ norms, const float* __restrict__ caches,
                                  float* __restrict__ out) {
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n_terms) return;
  const int t = (int)warp, f = term_field[t];
  const uint8_t* nrm = norms[f];
  const float* cache = caches + f * 256;
  float m = 0.0f;
  for (int64_t p = term_off[t] + lane; p < term_off[t + 1]; p += 32) {
    float freq = (float)f8[p];
    if (f8[p] == 255) {
      int a = 0, b = n_exc;
      while (a < b) { const int mid = (a + b) >> 1; if (exc_pos[mid] < p) a = mid + 1; else b = mid; }
      if (a < n_exc && exc_pos[a] == p) freq = (float)exc_freq[a];
    }
    m = fmaxf(m, __fmul_rn(freq, cache[nrm ? nrm[docs[p]] : 1]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) out[t] = m;
}

// 2-bit planes: four docs per byte, min(tf, 3) each
__global__ void plane_pack2_kernel(const uint8_t* __restrict__ planes, int64_t n_bytes_out, uint8_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_bytes_out) return;
  const uchar4 b = reinterpret_cast<const uchar4*>(planes)[i];
  out[i] = (uint8_t)(min((int)b.x, 3) | (min((int)b.y, 3) << 2) | (min((int)b.z, 3) << 4) | (min((int)b.w, 3) << 6));
}

// dense tf plane of one term: plane[doc] = min(freq, 255) for every posting of the term (the plane is zeroed first)
__global__ void plane_fill_kernel(const int32_t* __restrict__ docs, const uint8_t* __restrict__ f8, int64_t n,
                                  uint8_t* __restrict__ plane) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) plane[docs[i]] = f8[i];
}

// index-time skip data: for every term with a long list, the number of its postings below each granule boundary
struct GranTabLaunch {
  const int32_t* post_docs;
  const int64_t* row_off;   // [n_rows] first posting of the row's term
  const int32_t* row_n;     // [n_rows] postings of the row's term
  int32_t n_rows, n_gran, n_docs;
  uint32_t* tab;            // [n_rows][n_gran + 1]
};

__global__ void gran_table_kernel(GranTabLaunch G) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)G.n_rows * (G.n_gran + 1)) return;
  const int r = (int)(i / (G.n_gran + 1)), g = (int)(i % (G.n_gran + 1));
  const int64_t target64 = (int64_t)g << v3::kLogGran;
  const int32_t target = target64 > (int64_t)G.n_docs ? G.n_docs : (int32_t)target64;
  const int32_t* docs = G.post_docs + G.row_off[r];
  int lo = 0, hi = G.row_n[r];
  while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(docs + mid) < target) lo = mid + 1; else hi = mid; }
  G.tab[i] = (uint32_t)lo;
}

namespace {

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0, cap = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t count) {   // keeps the allocation when it is already large enough (workspace reuse)
    n = count;
    if (count <= cap) return NRTGPU_OK;
    if (p) { cudaFree(p); p = nullptr; cap = 0; }
    NRT_CUDA_TRY(cudaMalloc((void**)&p, count * sizeof(T)));
    cap = count;
    return NRTGPU_OK;
  }
  int upload_async(const T* h, size_t count, cudaStream_t st) {
    int rc = alloc(count);
    if (rc) return rc;
    if (count) NRT_CUDA_TRY(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, st));
    return NRTGPU_OK;
  }
  int upload(const T* h, size_t count) {
    int rc = alloc(count);
    if (rc) return rc;
    if (count) NRT_CUDA_TRY(cudaMemcpy(p, h, count * sizeof(T), cudaMemcpyHostToDevice));
    return NRTGPU_OK;
  }
  size_t bytes() const { return n * sizeof(T); }
};

}  // namespace

// A keyword column of an image (nrtgpu_index_add_keyword_columns): its term dictionary on the host, and on the device the
// bucket code 2i + 2 of ordinal i (0: no value) per doc (SORTED) or per value with the doc offsets (SORTED_SET, counted by
// the kMulti kernel instantiations: agg_collect_values)
struct KeywordColumn {
  int32_t n_terms = 0;
  bool multi = false;
  int64_t n_values = 0;               // length of codes
  std::vector<uint8_t> bytes;         // the dictionary: term t is bytes[off[t], off[t + 1])
  std::vector<int64_t> off;
  DevBuf<uint32_t> codes;             // [n_values]
  DevBuf<int64_t> doc_off;            // SORTED_SET: [n_docs + 1]
};

struct nrtgpu_ctx {
  int device = 0;
  std::mutex hyb_mu;             // O(k) hybrid stages share one pooled device scratch (no cudaMalloc per call)
  DevBuf<int32_t> hyb_scratch;
  PlanKnobs plan;                // the work planner's knobs, with the device's SM count
  int probe_cfg = 0;            // NRTGPU_PROBE_CFG: 0 auto, 1 always A (3 CTAs / SM), 2 always B (4 CTAs / SM)
  bool debug_modes = false;     // NRTGPU_DEBUG_MODES=1: per-launch kernel statistics on stderr (adds a stream synchronisation)
};

// which launch configuration of the probe kernel a launch takes (see probe_kernel.cuh kCtasA / kCtasB)
static inline bool ix_ctx_probe_cfg(const nrtgpu_ctx* c, bool visits_everything) { return c->probe_cfg == 2 || (c->probe_cfg == 0 && visits_everything); }

struct nrtgpu_index {
  nrtgpu_ctx* ctx = nullptr;
  int32_t n_docs = 0, doc_base = 0, n_terms = 0, n_fields = 0, n_columns = 0;
  // host-side dictionary
  std::vector<int64_t> term_off;
  std::vector<int32_t> term_field;
  std::vector<int64_t> term_df;
  std::vector<float> term_max_x;
  std::vector<int32_t> term_plane;   // dense tf plane per term, -1 for all but the densest terms
  std::vector<int32_t> term_gran;    // row of the granule offset table per term, -1 for short lists
  std::vector<int64_t> field_doc_count, field_sum_ttf;
  std::vector<uint8_t> field_has_norms;
  std::vector<float> field_k1, field_b;
  // device image
  DevBuf<int32_t> post_docs;
  DevBuf<uint8_t> post_f8;
  DevBuf<int64_t> exc_pos;
  DevBuf<int32_t> exc_freq;
  int64_t sum_freq = 0;             // sum of the exact freqs: the positions nrtgpu_index_add_positions expects
  bool has_positions = false;
  DevBuf<int32_t> positions;        // term positions, posting after posting (nrtgpu_index_add_positions)
  DevBuf<uint32_t> pos_off;         // [P] first position of each posting, relative to its term's base
  DevBuf<int64_t> pos_base;         // [n_terms + 1] first position of each term
  std::vector<int64_t> h_pos_base;  // ... its host copy (the multi-phrase unions' positions cap)
  DevBuf<uint32_t> parent_bits;     // the parent docs of the image's blocks (nrtgpu_index_add_parents)
  bool has_parents = false;
  int64_t n_parents = 0;
  std::vector<std::unique_ptr<DevBuf<uint8_t>>> norms;
  DevBuf<const uint8_t*> norms_ptrs;
  DevBuf<float> caches;
  DevBuf<uint32_t> gran_tab;        // [n_rows][n_gran + 1] index-time granule offsets (skip data) of the long lists
  int32_t gran_n = 0;
  DevBuf<uint8_t> dense_tf;         // [n_planes][dense_stride]: direct-address tf bytes of the densest terms
  DevBuf<uint8_t> dense_tf2;        // [n_planes][dense_stride / 4]: the same planes at 2 bits per doc (min(tf, 3))
  int64_t dense_stride = 0;
  int32_t n_planes = 0;
  DevBuf<uint8_t> field_min_norm;   // smallest non-zero norm byte per field (0 byte = doc lacks the field)
  std::vector<std::unique_ptr<DevBuf<int64_t>>> col64;
  std::vector<std::unique_ptr<DevBuf<int32_t>>> col32;
  std::vector<std::unique_ptr<DevBuf<uint8_t>>> col_has;
  std::vector<std::unique_ptr<DevBuf<uint32_t>>> col_code;      // per column: order-preserving sort code per doc (sort_kernel.cuh)
  std::vector<std::unique_ptr<DevBuf<uint64_t>>> col_distinct;  // per column: sorted distinct values (sortable domain)
  std::vector<int32_t> col_n_distinct;
  DevBuf<const int64_t*> col64_ptrs;
  DevBuf<const int32_t*> col32_ptrs;
  DevBuf<const uint8_t*> col_has_ptrs;
  std::vector<std::unique_ptr<DevBuf<int64_t>>> colmv_off;   // multi-valued columns: per-doc offsets (values sit in col64)
  DevBuf<const int64_t*> colmv_off_ptrs, colmv_val_ptrs;
  std::vector<uint8_t> col_multi;                            // [n_columns] 1 = multi-valued
  std::vector<std::unique_ptr<KeywordColumn>> kw;            // keyword columns (nrtgpu_index_add_keyword_columns)
  std::vector<int32_t> kw_n_terms;
  DevBuf<const uint32_t*> kw_code_ptrs;                      // [kw] the columns' codes, for the keyword clauses of DevIndexView
  DevBuf<const int64_t*> kw_off_ptrs;                        // [kw] SORTED_SET doc offsets, NULL for SORTED
  bool kw_added = false;
  DevBuf<uint32_t> live_bits;
  // vectors
  int32_t vec_dims = 0, vec_sim = 0, vec_count = 0;
  bool vec_is_byte = false;   // byte vector field (ByteVectorFieldDef): same image, byte score mapping
  DevBuf<float> vectors;
  DevBuf<__nv_bfloat16> vec_bf16;   // bf16 copy of the corpus for the tensor-core candidate stage (dims % 8 == 0)
  CUtensorMap vec_tmap;             // TMA tensor map over vec_bf16 (boxes of one GEMM corpus tile)
  DevBuf<float2> vec_ab;            // per-vector (a, b) of the approximate score a * dot + b
  bool vec_tc = false;
  float vec_dmax = 0.0f;    // largest vector magnitude (error bound of the kNN candidate-stage certificate)
  int32_t knn_last_uncertified = 0;   // queries of the last kNN call that took the exact fallback
  int32_t knn_last_gather = 0;        // queries of the last filtered kNN call scored over their filter's docs only
  float knn_last_filter_ms = 0.0f;    // device time of its filter evaluation
  cudaEvent_t knn_ev[2] = {};         // ... between these two events
  bool vec_docs_ascending = true;     // one vector per doc, ordinals in doc order (what the gather path's list sizes assume)
  DevBuf<float> vec_norm2;  // per-vector squared magnitude (double-accumulated, stored float) for cosine
  DevBuf<int32_t> vec_docs;
  int64_t device_bytes = 0;
  // reusable batch workspaces of the one-shot entry point (nrtgpu_search_bool), one per concurrent caller
  std::mutex ws_mu;
  std::mutex knn_mu;          // one kNN call at a time per index: they share knn_scratch
  std::mutex fetch_mu;        // fetch-phase scratch
  DevBuf<int32_t> f_cols, f_docs; DevBuf<int64_t> f_vals; DevBuf<uint8_t> f_has;
  KnnScratch knn_scratch;
  std::vector<nrtgpu_batch*> ws_free;
  ~nrtgpu_index();

  DevIndexView view() const {
    DevIndexView v;
    v.n_docs = n_docs; v.doc_base = doc_base;
    v.post_docs = post_docs.p; v.post_f8 = post_f8.p;
    v.exc_pos = exc_pos.p; v.exc_freq = exc_freq.p; v.n_exc = (int32_t)exc_pos.n;
    v.norms = norms_ptrs.p; v.caches = caches.p;
    v.col64 = col64_ptrs.p; v.col32 = col32_ptrs.p; v.col_has = col_has_ptrs.p;
    v.colmv_off = colmv_off_ptrs.p; v.colmv_val = colmv_val_ptrs.p;
    v.live_bits = live_bits.p;
    v.dense_tf = dense_tf.p; v.dense_stride = dense_stride; v.dense_tf2 = dense_tf2.p;
    v.gran_tab = gran_tab.p; v.n_gran = gran_n;
    v.positions = positions.p; v.pos_off = pos_off.p; v.pos_base = pos_base.p;
    v.kw_codes = kw_code_ptrs.p; v.kw_off = kw_off_ptrs.p;
    return v;
  }
  PlanDict dict() const {   // what batch compilation and planning read
    PlanDict d;
    d.n_docs = n_docs; d.doc_base = doc_base; d.n_terms = n_terms; d.n_columns = n_columns;
    d.term_off = term_off.data(); d.term_field = term_field.data(); d.term_df = term_df.data(); d.term_max_x = term_max_x.data();
    d.term_plane = term_plane.data(); d.term_gran = term_gran.data(); d.field_doc_count = field_doc_count.data();
    d.col_multi = col_multi.data(); d.col_n_distinct = col_n_distinct.data(); d.has_deletes = live_bits.p != nullptr;
    d.has_positions = has_positions;
    d.n_keyword = (int32_t)kw.size(); d.kw_n_terms = kw_n_terms.data();
    d.term_pos = has_positions ? h_pos_base.data() : nullptr;
    d.max_union_postings = ctx->plan.union_postings;
    d.has_parents = has_parents; d.n_parents = n_parents; d.max_join_children = ctx->plan.join_children;
    return d;
  }
  KnnCorpus knn_corpus() const {   // what the kNN stages read; NRTGPU_KNN_SIMT, read on every call, forces the fp32 SIMT stage
    const bool t = vec_tc && getenv("NRTGPU_KNN_SIMT") == nullptr;
    return {vectors.p, vec_norm2.p, vec_docs.p, vec_count, vec_dims, vec_sim | (vec_is_byte ? kKnnByteFlag : 0), doc_base, n_docs,
            live_bits.p, vec_dmax, t ? vec_bf16.p : nullptr, t ? &vec_tmap : nullptr, t ? vec_ab.p : nullptr};
  }
};

// a Sort of several fields ranked over one image (sort_kernel.cuh, sort_order_build)
struct nrtgpu_sort_order {
  const nrtgpu_index* ix = nullptr;
  int32_t n_fields = 0;
  bool score_first = false; int32_t score_reverse = 0;
  int32_t n_rank = 0;                   // fields of the rank: after the leading SCORE, up to the first DOCID inclusive
  SortFieldDev f[kMaxSortFields] = {};  // every field of the Sort (device pointers into the image)
  nrtgpu_sort_field spec[kMaxSortFields] = {};   // the Sort as given (orders of the leaves of one searcher must agree)
  DevBuf<int32_t> perm;                 // position -> doc
  DevBuf<uint32_t> rank;                // doc -> position + 1
};

// Where the additional collectors of a run count (cb.aggs, cb.nested): per aggregation its count table [nq][n_buckets]
// (terms) or metric words [nq] (min / max / sum), the bucket codes of its column and the distinct values they number; per
// nested min / max / sum collector its words [nq][n_buckets of the parent]. A single image fills it from the batch's own
// buffers and the image's columns on every run; a searcher points the batches of all its leaves at one set of reader-wide
// tables, each with that leaf's codes (agg_shared).
struct AggTables {
  unsigned int* counts[kMaxAggs];
  unsigned long long* dvals[kMaxAggs];
  const uint32_t* codes[kMaxAggs];
  const int64_t* offsets[kMaxAggs];   // SORTED_SET keyword terms: the doc offsets of codes (NULL: one code per doc)
  int32_t n_buckets[kMaxAggs];
  const uint64_t* distinct[kMaxAggs];  // NULL for keyword terms: bucket keys are ordinals
  unsigned long long* nest_words[kMaxAggs * kMaxNested];
};

struct nrtgpu_batch {
  nrtgpu_index* ix = nullptr;
  int32_t nq = 0, top_k = 0;
  CompiledBatch cb;            // host copies the async uploads read, kept until the next compilation
  WorkPlan plan;               // (search batches only)
  DevBuf<uint32_t> sbounds;            // probe kernel: [nq][4][n_slices * parts_max + 3] boundary posting offsets (batch_plan.h)
  DevBuf<v3::DevProbeQuery> pquery;    // probe kernel: [nq] per-query records (probe_query_kernel)
  DevBuf<unsigned int> work_counter;   // probe kernel: queue heads [2]
  DevBuf<unsigned long long> probe_stats;
  DevBuf<DevClause> clauses;
  DevBuf<DevQuery> queries;
  DevBuf<DevNode> nodes;          // tree batches: cb.nodes
  DevBuf<int32_t> node_begin;     // tree batches: cb.node_begin
  DevBuf<DevPhrase> phrases;      // tree batches: cb.phrases
  DevBuf<int32_t> phrase_begin;   // tree batches: cb.phrase_begin
  DevBuf<int32_t> work_query, work_slice;
  // multi-phrase unions of the batch (union_kernel.cuh), rebuilt by every batch_build that has some: the alternatives, the
  // sort's keys and values (double buffers), the run heads and their scan, the entries and their positions
  DevBuf<int64_t> u_alt_gstart, u_alt_post;
  DevBuf<int32_t> u_alt_term, u_alt_union, u_alt_field, u_clause;
  DevBuf<float> u_alt_weight;
  DevBuf<uint8_t> u_mode, u_temp;
  DevBuf<uint64_t> u_keys[2];
  DevBuf<int32_t> u_vals[2], u_head, u_incl, u_docs, u_first, u_npos, u_pos_off, u_positions;
  DevBuf<float> u_score;
  UnionView u_view = {};
  int64_t u_gathered = 0;         // the union postings gathered: the join entries start there in u_docs / u_score
  // block joins of the batch (join_kernel.cuh), rebuilt by every batch_build that has some: the child pass's work items,
  // the joins' modes and clauses, the emitted keys and scores (double buffers), the run heads and their scan
  DevBuf<int32_t> j_work_query, j_work_slice, j_clause, j_head, j_incl;
  DevBuf<uint8_t> j_mode, j_temp;
  DevBuf<uint64_t> j_keys[2];
  DevBuf<float> j_scores[2];
  DevBuf<unsigned int> j_count;
  DevBuf<int32_t> pruned;    // [nq] relation GTE flags
  DevBuf<int32_t> terminated; // [nq] terminateAfter cut the query short
  DevBuf<int32_t> timed_out;  // [nq] a work item of the query was skipped because the deadline had passed
  DevBuf<unsigned long long> clock0;  // [1] %globaltimer when the first work item of the run started
  std::vector<int32_t> h_flags;
  // sort-by-field (TopFieldCollector)
  int32_t sort_kind = 0, sort_column = 0, sort_reverse = 0;
  int64_t sort_missing_value = 0;
  DevBuf<int64_t> after_values; DevBuf<int32_t> after_docs; DevBuf<uint32_t> sort_missing_code;
  DevBuf<int64_t> out_sort_values;
  std::vector<int32_t> h_after_docs;
  const nrtgpu_sort_order* order = nullptr;   // nrtgpu_search_sorted_fields: the Sort's order (sort_kind COLUMN or kSortScoreRank)
  // additional collectors (aggregations, cb.aggs)
  DevBuf<unsigned int> agg_counts[kMaxAggs];
  DevBuf<unsigned long long> agg_dvals[kMaxAggs];
  DevBuf<AggLaunch> agg_launch;
  AggTables agg_tab = {};      // the tables of the current run (agg_shared: set by the searcher, not reset by the run)
  bool agg_shared = false;
  DevBuf<int64_t> agg_keys; DevBuf<int32_t> agg_cnts, agg_n, agg_tot; DevBuf<long long> agg_other;
  // nested collectors (cb.nested): [nq][n_buckets] words of the min / max / sum ones (pass 1), the selection's returned
  // buckets and slot map, and the top-hits run's key buffers (pass 2)
  DevBuf<unsigned long long> nest_words[kMaxAggs * kMaxNested];
  DevBuf<int32_t> agg_bucket, nest_slot; DevBuf<double> nest_vals;
  DevBuf<uint64_t> nest_keys; DevBuf<long long> nest_off; DevBuf<unsigned int> nest_fill;
  DevBuf<int32_t> nest_docs, nest_hcounts; DevBuf<float> nest_scores;
  // sorted top hits: FieldDoc values of the results; over several leaves the group's packed sorted records (leaves', then
  // merged) and the key scores of a leaf's selection
  DevBuf<int64_t> nest_svals, nest_rec; DevBuf<float> nest_rscores;
  // a searcher's leaf: per cb.nested entry, the leaf -> union maps of its Sort's keyword fields (empty: a single image)
  std::vector<std::array<const uint32_t*, kMaxSortFields>> nest_kw_map;
  DevBuf<AggLaunch> nest_launch;
  DevBuf<unsigned long long> p2_total; DevBuf<int32_t> p2_flags;   // the top-hits run's totalHits / pruned / terminated
  // filter collectors (cb.agg_filters): one row per FILTER aggregation on this image (agg_rows), built by batch_filter_rows
  // from the compiled filter queries (agg_fq) and the sorted value sets (agg_set), with the term bitmaps in agg_scratch (not
  // the index's kNN scratch, which a concurrent kNN call owns); agg_gate[i]: the row that gates aggregation i, NULL: none
  std::unique_ptr<nrtgpu_batch> agg_fq;
  KnnScratch agg_scratch;
  DevBuf<uint32_t> agg_rows; DevBuf<int64_t> agg_set;
  const uint32_t* agg_gate[kMaxAggs] = {};
  // the codes aggregation i counts through in the current run: its column's (agg_tab.codes), or, under a row, agg_row_codes_kernel's
  DevBuf<uint32_t> agg_fcodes[kMaxAggs];
  const uint32_t* agg_codes[kMaxAggs] = {};
  // second pass of QueryRescorer (nrtgpu_score_docs / nrtgpu_rescore_query)
  DevBuf<int32_t> sd_docs, sd_counts; DevBuf<uint8_t> sd_match; DevBuf<float> sd_scores, sd_first;
  bool limits_active = false, disallow_partial = false;
  double timeout_sec = 0.0;
  long long deadline_ns = 0;       // budget from the first work item on (0: none)
  int64_t ta_scalar = 0;           // terminateAfter (0: none)
  int64_t terminate_after_max_recall = 0;
  DevBuf<unsigned long long> known_hits;        // probe kernel: plan.known_hits
  DevBuf<int32_t> warm_exact;                   // probe kernel: plan.warm_exact
  DevBuf<uint64_t> theta;
  DevBuf<unsigned long long> total_hits;
  DevBuf<uint64_t> slice_keys;
  DevBuf<int32_t> slice_cnt;
  DevBuf<int32_t> out_docs;
  DevBuf<float> out_scores;
  DevBuf<int32_t> out_counts;
  static constexpr int kEvRing = 64;
  cudaEvent_t ev[kEvRing][3] = {};
  int runs_recorded = 0;   // since the last timing reset
  bool ran = false;
  // optional caller-provided device output buffers (e.g. torch tensors feeding the NCCL all-gather)
  int32_t* bound_docs = nullptr; float* bound_scores = nullptr; int32_t* bound_counts = nullptr;
  long long* bound_total = nullptr; int32_t* bound_flags = nullptr;   // packed record (nrtgpu_batch_bind_packed)
  int64_t* bound_values = nullptr;   // sorted record (batch_bind_sorted): FieldDoc values
  int32_t* o_docs() { return bound_docs ? bound_docs : out_docs.p; }
  float* o_scores() { return bound_scores ? bound_scores : out_scores.p; }
  int32_t* o_counts() { return bound_counts ? bound_counts : out_counts.p; }
  int64_t* o_sort_values() { return bound_values ? bound_values : out_sort_values.p; }
  void unbind() {
    bound_docs = nullptr; bound_scores = nullptr; bound_counts = nullptr; bound_total = nullptr; bound_flags = nullptr; bound_values = nullptr;
  }
  ~nrtgpu_batch() { for (auto& r : ev) for (auto& e : r) if (e) cudaEventDestroy(e); }
};

// index-time impacts: max over a term's postings of tf * cache[norm]; depends on the index-wide avgdl through cache[]
static int compute_term_max_x(nrtgpu_index* ix) {
  ix->term_max_x.assign((size_t)ix->n_terms, 0.0f);
  const int64_t P = ix->n_terms ? ix->term_off[(size_t)ix->n_terms] : 0;
  if (P <= 0) return NRTGPU_OK;
  int rc;
  DevBuf<int64_t> d_off; DevBuf<int32_t> d_tf; DevBuf<float> d_mx;
  if ((rc = d_off.upload(ix->term_off.data(), ix->term_off.size()))) return rc;
  if ((rc = d_tf.upload(ix->term_field.data(), ix->term_field.size()))) return rc;
  if ((rc = d_mx.alloc((size_t)ix->n_terms))) return rc;
  const int64_t threads = (int64_t)ix->n_terms * 32;
  term_max_x_kernel<<<(unsigned)((threads + 255) / 256), 256>>>(d_off.p, ix->n_terms, d_tf.p, ix->post_docs.p, ix->post_f8.p,
                                                                 ix->exc_pos.p, ix->exc_freq.p, (int)ix->exc_pos.n, ix->norms_ptrs.p,
                                                                 ix->caches.p, d_mx.p);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpy(ix->term_max_x.data(), d_mx.p, (size_t)ix->n_terms * sizeof(float), cudaMemcpyDeviceToHost));
  return NRTGPU_OK;
}

static int upload_live_docs(nrtgpu_index* ix, const uint8_t* live_docs) {
  if (!live_docs) { ix->live_bits.n = 0; if (ix->live_bits.p) { cudaFree(ix->live_bits.p); ix->live_bits.p = nullptr; ix->live_bits.cap = 0; } return NRTGPU_OK; }
  std::vector<uint32_t> bits(((size_t)ix->n_docs + 31) / 32, 0u);
  for (int32_t i = 0; i < ix->n_docs; ++i) if (live_docs[i]) bits[(size_t)i >> 5] |= 1u << (i & 31);
  return ix->live_bits.upload(bits.data(), bits.size());
}
nrtgpu_index::~nrtgpu_index() {
  for (auto* b : ws_free) delete b;
  for (auto e : knn_ev) if (e) cudaEventDestroy(e);
}

extern "C" {

const char* nrtgpu_last_error(void) { return g_last_error.c_str(); }
int nrtgpu_version(void) { return 1; }

int nrtgpu_init(int device_id, nrtgpu_ctx** out) {
  if (!out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_init: out is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    NRT_FAIL(NRTGPU_ERR_CUDA, std::string("nrtgpu_init: no CUDA device (") + cudaGetErrorString(e) +
                                  "); this engine has no CPU fallback");
  if (device_id < 0 || device_id >= n) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_init: bad device id");
  NRT_CUDA_TRY(cudaSetDevice(device_id));
  cudaDeviceProp prop;
  NRT_CUDA_TRY(cudaGetDeviceProperties(&prop, device_id));
  if (prop.major != 9 || prop.minor != 0) NRT_FAIL(NRTGPU_ERR_CUDA, "nrtgpu_init: device is not sm_90 (kernels are built for sm_90a only)");
  std::unique_ptr<nrtgpu_ctx> c(new nrtgpu_ctx);   // released to the caller only when every attribute call succeeded
  c->device = device_id;
  c->plan.sm_count = prop.multiProcessorCount;
  c->debug_modes = getenv("NRTGPU_DEBUG_MODES") != nullptr;
  { const char* e = getenv("NRTGPU_PROBE_CFG"); c->probe_cfg = e ? atoi(e) : 0; }
  { const char* e = getenv("NRTGPU_WARM_MIN_DOCS"); if (e && atoll(e) > 0) c->plan.warm_min_docs = atoll(e); }
  { const char* e = getenv("NRTGPU_SLICE_GRAN"); if (e && atoi(e) >= 64) c->plan.slice_gran = std::min(atoi(e), (int)v3::kMaxSliceGran); }
  { const char* e = getenv("NRTGPU_ITEM_POSTINGS"); if (e && atoll(e) > 0) c->plan.item_postings = atoll(e); }
  { const char* e = getenv("NRTGPU_ITEM_SHARE"); if (e && atoll(e) > 0) c->plan.item_share = atoll(e); }
  { const char* e = getenv("NRTGPU_ITEM_SHARE_FULL"); if (e && atoll(e) > 0) c->plan.item_share_full = atoll(e); }
  { const char* e = getenv("NRTGPU_UNION_POSTINGS"); if (e && atoll(e) > 0) c->plan.union_postings = std::min<int64_t>(atoll(e), kMaxUnionPostings); }
  { const char* e = getenv("NRTGPU_JOIN_CHILDREN"); if (e && atoll(e) > 0) c->plan.join_children = std::min<int64_t>(atoll(e), kMaxJoinChildren); }
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmem)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_union_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmemU)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_union_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmemU)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_union_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmemU)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(bool_window_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BoolTreeSmemU)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(v3::posting_probe_kernel<false, false, v3::kCtasA, v3::kStageA, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)sizeof(v3::ProbeSmemT<v3::kStageA>)));
  NRT_CUDA_TRY(cudaFuncSetAttribute(v3::posting_probe_kernel<false, false, v3::kCtasB, v3::kStageB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)sizeof(v3::ProbeSmemT<v3::kStageB>)));
#define NRT_PROBE_ATTR(S, D) \
  NRT_CUDA_TRY(cudaFuncSetAttribute(v3::posting_probe_kernel<S, D, v3::kCtasA, v3::kStageA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(v3::ProbeSmemT<v3::kStageA>))); \
  NRT_CUDA_TRY(cudaFuncSetAttribute(v3::posting_probe_kernel<S, D, v3::kCtasB, v3::kStageB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(v3::ProbeSmemT<v3::kStageB>)));
  NRT_PROBE_ATTR(true, false) NRT_PROBE_ATTR(false, false) NRT_PROBE_ATTR(true, true) NRT_PROBE_ATTR(false, true)
#undef NRT_PROBE_ATTR
  NRT_CUDA_TRY(cudaFuncSetAttribute(tc::knn_gemm_bf16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::kGemmSmem));
  NRT_CUDA_TRY(cudaFuncSetAttribute(tc::knn_gemm_bf16_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::kGemmSmem));
  *out = c.release();
  return NRTGPU_OK;
}

void nrtgpu_shutdown(nrtgpu_ctx* ctx) { delete ctx; }

int nrtgpu_index_build(nrtgpu_ctx* ctx, const nrtgpu_shard_desc* d, nrtgpu_index** out) {
  if (!ctx || !d || !out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: NULL argument");
  if (d->n_docs < 0 || d->n_terms < 0 || d->n_fields < 0 || d->n_columns < 0)
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: negative size");
  if (d->n_terms > 0 && (!d->term_off || d->n_fields < 1 || !d->field_doc_count || !d->field_sum_ttf))
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: terms need term_off and field statistics");
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  std::unique_ptr<nrtgpu_index> ix(new nrtgpu_index);
  ix->ctx = ctx;
  ix->n_docs = d->n_docs; ix->doc_base = d->doc_base; ix->n_terms = d->n_terms;
  ix->n_fields = d->n_fields; ix->n_columns = d->n_columns;
  int rc;
  const int64_t P = d->n_terms ? d->term_off[d->n_terms] : 0;
  ix->term_off.assign(d->term_off, d->term_off + (d->n_terms ? d->n_terms + 1 : 0));
  ix->term_field.resize(d->n_terms);
  ix->term_df.resize(d->n_terms);
  for (int t = 0; t < d->n_terms; ++t) {
    int f = d->term_field ? d->term_field[t] : 0;
    if (f < 0 || f >= d->n_fields) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: term_field out of range");
    int64_t len = d->term_off[t + 1] - d->term_off[t];
    if (len < 0 || len > INT32_MAX) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: bad term_off");
    ix->term_field[t] = f;
    ix->term_df[t] = d->term_df ? d->term_df[t] : len;
  }
  if (d->n_terms > 0 && d->term_off[0] != 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: term_off[0] must be 0");
  if (P > 0 && (!d->post_docs || !d->post_freqs)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: NULL postings");
  // every list strictly ascending and inside [0, n_docs): the kernels binary-search the lists and index per-doc arrays with them
  for (int t = 0; t < d->n_terms; ++t) {
    int32_t prev = -1;
    for (int64_t p = d->term_off[t]; p < d->term_off[t + 1]; ++p) {
      const int32_t doc = d->post_docs[p];
      if (doc <= prev || doc >= d->n_docs) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: post_docs must be strictly ascending per term and < n_docs");
      prev = doc;
    }
  }
  if (d->vec_dims < 0 || d->vec_count < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: negative vector size");
  if (d->vec_dims > 0 && d->vec_count > 0) {
    if (!d->vec_docs && d->vec_count > d->n_docs) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: vec_count > n_docs with an identity ord -> doc map");
    if (d->vec_docs) for (int32_t i = 0; i < d->vec_count; ++i)
      if (d->vec_docs[i] < 0 || d->vec_docs[i] >= d->n_docs) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: vec_docs out of range");
  }
  ix->field_doc_count.assign(d->field_doc_count, d->field_doc_count + d->n_fields);
  ix->field_sum_ttf.assign(d->field_sum_ttf, d->field_sum_ttf + d->n_fields);
  // postings
  const size_t pad = (size_t)v3::kPostingPad;
  if ((rc = ix->post_docs.alloc((size_t)P + pad))) return rc;
  NRT_CUDA_TRY(cudaMemset(ix->post_docs.p, 0x7f, ((size_t)P + pad) * sizeof(int32_t)));
  if (P) NRT_CUDA_TRY(cudaMemcpy(ix->post_docs.p, d->post_docs, (size_t)P * sizeof(int32_t), cudaMemcpyHostToDevice));
  {
    std::vector<uint8_t> f8((size_t)P + pad, 0);
    std::vector<int64_t> epos; std::vector<int32_t> efreq;
    for (int64_t p = 0; p < P; ++p) {
      int32_t f = d->post_freqs[p];
      if (f < 1) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: term frequency < 1");
      ix->sum_freq += f;
      if (f >= 255) { f8[(size_t)p] = 255; epos.push_back(p); efreq.push_back(f); } else f8[(size_t)p] = (uint8_t)f;
    }
    if ((rc = ix->post_f8.upload(f8.data(), (size_t)P + pad))) return rc;
    if ((rc = ix->exc_pos.upload(epos.data(), epos.size()))) return rc;
    if ((rc = ix->exc_freq.upload(efreq.data(), efreq.size()))) return rc;
  }
  // dense tf planes (plan_planes)
  {
    std::vector<int32_t> dense_terms;
    const int64_t stride = plan_planes(d->n_docs, d->n_terms, d->term_off, ix->term_plane, dense_terms);
    if (!dense_terms.empty()) {
      ix->dense_stride = stride; ix->n_planes = (int32_t)dense_terms.size();
      if ((rc = ix->dense_tf.alloc((size_t)stride * dense_terms.size()))) return rc;
      NRT_CUDA_TRY(cudaMemset(ix->dense_tf.p, 0, ix->dense_tf.bytes()));
      for (size_t k = 0; k < dense_terms.size(); ++k) {
        const int32_t t = dense_terms[k];
        const int64_t off = d->term_off[t], n = d->term_off[t + 1] - off;
        plane_fill_kernel<<<(unsigned)((n + 255) / 256), 256>>>(ix->post_docs.p + off, ix->post_f8.p + off, n,
                                                                 ix->dense_tf.p + (size_t)k * stride);
      }
      NRT_CUDA_TRY(cudaGetLastError());
      const int64_t n2 = (int64_t)(stride / 4) * (int64_t)dense_terms.size();
      if ((rc = ix->dense_tf2.alloc((size_t)n2))) return rc;
      plane_pack2_kernel<<<(unsigned)((n2 + 255) / 256), 256>>>(ix->dense_tf.p, n2, ix->dense_tf2.p);
      NRT_CUDA_TRY(cudaGetLastError());
    }
  }
  // skip data (plan_gran_rows)
  {
    std::vector<int64_t> row_off; std::vector<int32_t> row_n;
    const int32_t n_gran = plan_gran_rows(d->n_docs, d->n_terms, d->term_off, ix->term_gran, row_off, row_n);
    ix->gran_n = n_gran;
    if (!row_off.empty()) {
      DevBuf<int64_t> d_ro; DevBuf<int32_t> d_rn;
      if ((rc = d_ro.upload(row_off.data(), row_off.size()))) return rc;
      if ((rc = d_rn.upload(row_n.data(), row_n.size()))) return rc;
      const int64_t total = (int64_t)row_off.size() * (n_gran + 1);
      if ((rc = ix->gran_tab.alloc((size_t)total))) return rc;
      GranTabLaunch G;
      G.post_docs = ix->post_docs.p; G.row_off = d_ro.p; G.row_n = d_rn.p; G.n_rows = (int32_t)row_off.size();
      G.n_gran = n_gran; G.n_docs = d->n_docs; G.tab = ix->gran_tab.p;
      gran_table_kernel<<<(unsigned)((total + 255) / 256), 256>>>(G);
      NRT_CUDA_TRY(cudaGetLastError());
      NRT_CUDA_TRY(cudaDeviceSynchronize());
    }
  }
  // norms + BM25 caches
  {
    std::vector<const uint8_t*> ptrs((size_t)d->n_fields, nullptr);
    std::vector<float> caches((size_t)d->n_fields * 256);
    std::vector<uint8_t> min_norm((size_t)d->n_fields, 1);
    ix->field_has_norms.resize(d->n_fields);
    for (int f = 0; f < d->n_fields; ++f) {
      ix->norms.emplace_back(new DevBuf<uint8_t>);
      const uint8_t* h = d->norms ? d->norms[f] : nullptr;
      ix->field_has_norms[f] = h != nullptr;
      if (h) {
        if ((rc = ix->norms.back()->upload(h, (size_t)d->n_docs))) return rc;
        ptrs[f] = ix->norms.back()->p;
        int mn = 256;
        for (int32_t i = 0; i < d->n_docs; ++i) if (h[i] != 0 && h[i] < mn) mn = h[i];
        min_norm[f] = (uint8_t)(mn == 256 ? 0 : mn);
      }
      float k1 = d->field_k1 ? d->field_k1[f] : 1.2f, b = d->field_b ? d->field_b[f] : 0.75f;
      ix->field_k1.push_back(k1); ix->field_b.push_back(b);
      int64_t dc = d->field_doc_count[f];
      float avgdl = dc > 0 ? (float)((double)d->field_sum_ttf[f] / (double)dc) : 1.0f;
      bm25_cache(k1, b, avgdl, &caches[(size_t)f * 256]);
    }
    if ((rc = ix->norms_ptrs.upload(ptrs.data(), ptrs.size()))) return rc;
    if ((rc = ix->caches.upload(caches.data(), caches.size()))) return rc;
    if ((rc = ix->field_min_norm.upload(min_norm.data(), min_norm.size()))) return rc;
  }
  // numeric doc-value columns (int32 when the value range allows: 4 B/doc gathers)
  {
    std::vector<const int64_t*> p64((size_t)d->n_columns, nullptr);
    std::vector<const int32_t*> p32((size_t)d->n_columns, nullptr);
    // (one more entry than columns, always NULL: the column a filter collector's aggregation names, a column without a has
    // array, so agg_collect counts it through its codes alone)
    std::vector<const uint8_t*> ph((size_t)d->n_columns + 1, nullptr);
    std::vector<const int64_t*> pmo((size_t)d->n_columns, nullptr), pmv((size_t)d->n_columns, nullptr);
    ix->col_multi.assign((size_t)d->n_columns, 0);
    for (int c = 0; c < d->n_columns; ++c) {
      ix->col64.emplace_back(new DevBuf<int64_t>);
      ix->col32.emplace_back(new DevBuf<int32_t>);
      ix->col_has.emplace_back(new DevBuf<uint8_t>);
      ix->colmv_off.emplace_back(new DevBuf<int64_t>);
      const int64_t* h = d->columns[c];
      if (!h) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: NULL column");
      const int64_t* mo = d->column_offsets ? d->column_offsets[c] : nullptr;
      if (mo) {   // SORTED_NUMERIC: CSR of values per doc
        if (mo[0] != 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: column_offsets[c][0] must be 0");
        for (int32_t i = 0; i < d->n_docs; ++i) {
          if (mo[i + 1] < mo[i]) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: column_offsets must be non-decreasing");
          for (int64_t p = mo[i] + 1; p < mo[i + 1]; ++p)
            if (h[p] < h[p - 1]) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: the values of a doc must be ascending (SortedNumericDocValues)");
        }
        ix->col_multi[(size_t)c] = 1;
        if ((rc = ix->colmv_off.back()->upload(mo, (size_t)d->n_docs + 1))) return rc;
        if ((rc = ix->col64.back()->upload(h, (size_t)std::max<int64_t>(mo[d->n_docs], 1)))) return rc;
        pmo[c] = ix->colmv_off.back()->p; pmv[c] = ix->col64.back()->p;
        continue;
      }
      bool fits = true;
      for (int32_t i = 0; i < d->n_docs; ++i) if (h[i] < INT32_MIN || h[i] > INT32_MAX) { fits = false; break; }
      if (fits) {
        std::vector<int32_t> tmp((size_t)d->n_docs);
        for (int32_t i = 0; i < d->n_docs; ++i) tmp[i] = (int32_t)h[i];
        if ((rc = ix->col32.back()->upload(tmp.data(), tmp.size()))) return rc;
        p32[c] = ix->col32.back()->p;
      } else {
        if ((rc = ix->col64.back()->upload(h, (size_t)d->n_docs))) return rc;
        p64[c] = ix->col64.back()->p;
      }
      const uint8_t* hh = d->column_has ? d->column_has[c] : nullptr;
      if (hh) { if ((rc = ix->col_has.back()->upload(hh, (size_t)d->n_docs))) return rc; ph[c] = ix->col_has.back()->p; }
    }
    // sort codes of every column (TopFieldCollector path): one device sort per column at build time
    if (d->n_columns > 0 && d->n_docs > 0) {
      DevBuf<uint64_t> keys; DevBuf<int32_t> idx, rank;
      if ((rc = keys.alloc((size_t)d->n_docs)) || (rc = idx.alloc((size_t)d->n_docs)) || (rc = rank.alloc((size_t)d->n_docs))) return rc;
      for (int c = 0; c < d->n_columns; ++c) {
        ix->col_code.emplace_back(new DevBuf<uint32_t>);
        ix->col_distinct.emplace_back(new DevBuf<uint64_t>);
        if (ix->col_multi[(size_t)c]) { ix->col_n_distinct.push_back(0); continue; }   // no sort / terms on a multi-valued column
        if ((rc = ix->col_code.back()->alloc((size_t)d->n_docs))) return rc;
        if ((rc = ix->col_distinct.back()->alloc((size_t)d->n_docs))) return rc;
        NRT_CUDA_TRY(cudaMemset(ix->col_code.back()->p, 0, ix->col_code.back()->bytes()));
        int32_t nd = 0;
        if ((rc = sort_codes_build(p64[c], p32[c], ph[c], d->n_docs, ix->col_code.back()->p, keys.p, idx.p, rank.p,
                                   ix->col_distinct.back()->p, &nd))) return rc;
        ix->col_n_distinct.push_back(nd);
      }
    }
    if ((rc = ix->col64_ptrs.upload(p64.data(), p64.size()))) return rc;
    if ((rc = ix->col32_ptrs.upload(p32.data(), p32.size()))) return rc;
    if ((rc = ix->col_has_ptrs.upload(ph.data(), ph.size()))) return rc;
    if ((rc = ix->colmv_off_ptrs.upload(pmo.data(), pmo.size()))) return rc;
    if ((rc = ix->colmv_val_ptrs.upload(pmv.data(), pmv.size()))) return rc;
  }
  // index-time impacts (list-wide score bounds for MAXSCORE)
  if ((rc = compute_term_max_x(ix.get()))) return rc;
  if (d->live_docs && (rc = upload_live_docs(ix.get(), d->live_docs))) return rc;
  // vectors
  if (d->vec_dims > 0 && d->vec_count > 0) {
    if (!d->vectors) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: NULL vectors");
    if (d->vec_element_type != NRTGPU_VEC_FLOAT32 && d->vec_element_type != NRTGPU_VEC_INT8) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: bad vec_element_type");
    if (d->vec_dims > 4096) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_build: vector dims > 4096 (VectorFieldDef.java:96)");
    ix->vec_dims = d->vec_dims; ix->vec_sim = d->vec_similarity; ix->vec_count = d->vec_count;
    ix->vec_is_byte = d->vec_element_type == NRTGPU_VEC_INT8;
    if (ix->vec_is_byte) {   // bytes are held as exact floats (every int8 is exact in fp32 and in bf16)
      const int8_t* src = reinterpret_cast<const int8_t*>(d->vectors);
      std::vector<float> tmp((size_t)d->vec_count * d->vec_dims);
      for (size_t i = 0; i < tmp.size(); ++i) tmp[i] = (float)src[i];
      if ((rc = ix->vectors.upload(tmp.data(), tmp.size()))) return rc;
    } else if ((rc = ix->vectors.upload(d->vectors, (size_t)d->vec_count * d->vec_dims))) return rc;
    if (d->vec_docs) { if ((rc = ix->vec_docs.upload(d->vec_docs, (size_t)d->vec_count))) return rc; }
    for (int32_t i = 1; d->vec_docs && i < d->vec_count; ++i) if (d->vec_docs[i] <= d->vec_docs[i - 1]) ix->vec_docs_ascending = false;
    if ((rc = ix->vec_norm2.alloc((size_t)d->vec_count))) return rc;
    if ((rc = knn_prepare_norms(ix->vectors.p, ix->vec_count, ix->vec_dims, ix->vec_norm2.p))) return rc;
    {
      DevBuf<unsigned int> d_mx;
      if ((rc = d_mx.alloc(1))) return rc;
      NRT_CUDA_TRY(cudaMemset(d_mx.p, 0, sizeof(unsigned int)));
      knn_max_norm2_kernel<<<256, 256>>>(ix->vec_norm2.p, ix->vec_count, d_mx.p);
      NRT_CUDA_TRY(cudaGetLastError());
      float mx = 0.0f;
      NRT_CUDA_TRY(cudaMemcpy(&mx, d_mx.p, sizeof(float), cudaMemcpyDeviceToHost));
      ix->vec_dmax = std::sqrt(mx) * 1.0001f;
    }
    if (d->vec_dims % 8 == 0) {   // TMA needs 16-byte row pitch
      if ((rc = ix->vec_bf16.alloc((size_t)d->vec_count * d->vec_dims))) return rc;
      tc::f32_to_bf16_kernel<<<1024, 256>>>(ix->vectors.p, ix->vec_bf16.p, (size_t)d->vec_count * d->vec_dims);
      NRT_CUDA_TRY(cudaGetLastError());
      if ((rc = tc::make_tensor_map_bf16(&ix->vec_tmap, ix->vec_bf16.p, (uint64_t)d->vec_count, (uint64_t)d->vec_dims, tc::BN))) return rc;
      if ((rc = ix->vec_ab.alloc((size_t)d->vec_count))) return rc;
      knn_ab_kernel<<<(d->vec_count + 255) / 256, 256>>>(ix->vec_norm2.p, d->vec_count, d->vec_similarity, ix->vec_ab.p);
      NRT_CUDA_TRY(cudaGetLastError());
      ix->vec_tc = true;
    }
  }
  ix->device_bytes = (int64_t)(ix->gran_tab.bytes() + ix->dense_tf.bytes() + ix->dense_tf2.bytes() + ix->post_docs.bytes() + ix->post_f8.bytes() + ix->exc_pos.bytes() + ix->exc_freq.bytes() +
                               ix->caches.bytes() + ix->live_bits.bytes() + ix->vectors.bytes() + ix->vec_norm2.bytes() +
                               ix->vec_docs.bytes() + ix->vec_bf16.bytes());
  for (auto& b : ix->norms) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->col64) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->col32) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->col_has) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->colmv_off) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->col_code) ix->device_bytes += (int64_t)b->bytes();
  for (auto& b : ix->col_distinct) ix->device_bytes += (int64_t)b->bytes();
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  *out = ix.release();
  return NRTGPU_OK;
}

int nrtgpu_index_close(nrtgpu_index* ix) {
  if (!ix) return NRTGPU_OK;
  cudaSetDevice(ix->ctx->device);
  delete ix;
  return NRTGPU_OK;
}

int64_t nrtgpu_index_device_bytes(const nrtgpu_index* ix) { return ix ? ix->device_bytes : 0; }

int nrtgpu_index_add_positions(nrtgpu_index* ix, const int32_t* positions, int64_t n_positions) {
  if (!ix || (n_positions > 0 && !positions)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_positions: NULL argument");
  if (n_positions != ix->sum_freq)
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_positions: n_positions must be the sum of the postings' freqs (" +
                                     std::to_string(ix->sum_freq) + "), not " + std::to_string(n_positions));
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  NRT_CUDA_TRY(cudaDeviceSynchronize());   // searches in flight on this image finish against the old positions
  // the exact freq of every posting (the saturated byte and the exception list) gives each posting's position range
  const int64_t P = ix->n_terms ? ix->term_off[(size_t)ix->n_terms] : 0;
  std::vector<uint8_t> f8((size_t)P);
  std::vector<int64_t> epos(ix->exc_pos.n); std::vector<int32_t> efreq(ix->exc_freq.n);
  if (P) NRT_CUDA_TRY(cudaMemcpy(f8.data(), ix->post_f8.p, (size_t)P, cudaMemcpyDeviceToHost));
  if (!epos.empty()) NRT_CUDA_TRY(cudaMemcpy(epos.data(), ix->exc_pos.p, epos.size() * sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (!efreq.empty()) NRT_CUDA_TRY(cudaMemcpy(efreq.data(), ix->exc_freq.p, efreq.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  std::vector<uint32_t> off((size_t)P);
  std::vector<int64_t> base((size_t)ix->n_terms + 1, 0);
  int64_t run = 0; size_t e = 0;
  for (int32_t t = 0; t < ix->n_terms; ++t) {
    base[(size_t)t] = run;
    for (int64_t p = ix->term_off[(size_t)t]; p < ix->term_off[(size_t)t + 1]; ++p) {
      int64_t f = f8[(size_t)p];
      if (f == 255) { while (e < epos.size() && epos[e] < p) ++e; if (e < epos.size() && epos[e] == p) f = efreq[e]; }
      if (run - base[(size_t)t] > (int64_t)UINT32_MAX) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nrtgpu_index_add_positions: more than 2^32 positions of one term");
      off[(size_t)p] = (uint32_t)(run - base[(size_t)t]);
      for (int64_t i = run; i < run + f; ++i) {
        if (positions[i] < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_positions: negative position");
        if (i > run && positions[i] < positions[i - 1]) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_positions: positions descend within a posting");
      }
      run += f;
    }
  }
  base[(size_t)ix->n_terms] = run;
  const int64_t old_bytes = (int64_t)(ix->positions.bytes() + ix->pos_off.bytes() + ix->pos_base.bytes());
  int rc;
  if ((rc = ix->positions.upload(positions, (size_t)n_positions))) return rc;
  if ((rc = ix->pos_off.upload(off.data(), off.size()))) return rc;
  if ((rc = ix->pos_base.upload(base.data(), base.size()))) return rc;
  ix->device_bytes += (int64_t)(ix->positions.bytes() + ix->pos_off.bytes() + ix->pos_base.bytes()) - old_bytes;
  ix->h_pos_base = std::move(base);
  ix->has_positions = true;
  return NRTGPU_OK;
}

int nrtgpu_index_add_parents(nrtgpu_index* ix, int32_t root_term) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_parents: NULL index");
  if (root_term < 0 || root_term >= ix->n_terms) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_parents: term id out of range");
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  NRT_CUDA_TRY(cudaDeviceSynchronize());   // searches in flight on this image finish against the old parents
  const int64_t old_bytes = (int64_t)ix->parent_bits.bytes();
  const size_t words = std::max<size_t>(((size_t)ix->n_docs + 31) / 32, 1);
  int rc;
  if ((rc = ix->parent_bits.alloc(words))) return rc;
  NRT_CUDA_TRY(cudaMemset(ix->parent_bits.p, 0, words * sizeof(uint32_t)));
  const int64_t p0 = ix->term_off[(size_t)root_term], np = ix->term_off[(size_t)root_term + 1] - p0;
  if (np > 0) parent_bits_kernel<<<(unsigned)((np + 255) / 256), 256>>>(ix->post_docs.p + p0, np, ix->parent_bits.p);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  ix->device_bytes += (int64_t)ix->parent_bits.bytes() - old_bytes;
  ix->n_parents = np;
  ix->has_parents = true;
  return NRTGPU_OK;
}

int nrtgpu_index_add_keyword_columns(nrtgpu_index* ix, const nrtgpu_keyword_column* cols, int32_t n) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_keyword_columns: NULL index");
  if (ix->kw_added) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_add_keyword_columns: the image already has its keyword columns");
  int rc;
  if ((rc = check_keyword_columns(ix->n_docs, cols, n))) return rc;
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  std::vector<std::unique_ptr<KeywordColumn>> kw;
  int64_t bytes = 0;
  for (int32_t k = 0; k < n; ++k) {   // built aside: a failure leaves the image as it was
    const nrtgpu_keyword_column& c = cols[k];
    std::unique_ptr<KeywordColumn> x(new KeywordColumn);
    x->n_terms = c.n_terms; x->multi = c.multi_valued != 0;
    x->n_values = x->multi ? c.doc_offsets[ix->n_docs] : ix->n_docs;
    x->off.assign(c.term_offsets, c.term_offsets + c.n_terms + 1);
    if (c.term_offsets[c.n_terms] > 0) x->bytes.assign(c.term_bytes, c.term_bytes + c.term_offsets[c.n_terms]);
    std::vector<uint32_t> code((size_t)x->n_values);
    for (int64_t v = 0; v < x->n_values; ++v) code[(size_t)v] = c.ords[v] < 0 ? 0u : 2u * (uint32_t)c.ords[v] + 2u;
    if ((rc = x->codes.alloc(std::max<size_t>(code.size(), 1)))) return rc;   // (one word at least: a column without values)
    if (!code.empty()) NRT_CUDA_TRY(cudaMemcpy(x->codes.p, code.data(), code.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    x->codes.n = code.size();
    if (x->multi && (rc = x->doc_off.upload(c.doc_offsets, (size_t)ix->n_docs + 1))) return rc;
    bytes += (int64_t)(x->codes.bytes() + x->doc_off.bytes());
    kw.push_back(std::move(x));
  }
  if (n > 0) {   // (no image reads these before kw_added is set)
    std::vector<const uint32_t*> cp; std::vector<const int64_t*> op;
    for (auto& x : kw) { cp.push_back(x->codes.p); op.push_back(x->multi ? x->doc_off.p : nullptr); }
    if ((rc = ix->kw_code_ptrs.upload(cp.data(), cp.size())) || (rc = ix->kw_off_ptrs.upload(op.data(), op.size()))) return rc;
  }
  ix->kw = std::move(kw);
  for (auto& x : ix->kw) ix->kw_n_terms.push_back(x->n_terms);
  ix->kw_added = true;
  ix->device_bytes += bytes;
  return NRTGPU_OK;
}

// the bytes of term `ord` of a host dictionary (bytes, off) into out (min(len, cap) of them), its length into *len
static void copy_term(const std::vector<uint8_t>& bytes, const std::vector<int64_t>& off, int32_t ord, uint8_t* out, int32_t cap,
                      int32_t* len) {
  const int64_t a = off[(size_t)ord], l = off[(size_t)ord + 1] - a;
  *len = (int32_t)l;
  if (out && cap > 0 && l > 0) std::memcpy(out, bytes.data() + a, (size_t)std::min<int64_t>(l, cap));
}

int nrtgpu_index_keyword_seek(const nrtgpu_index* ix, int32_t column, const uint8_t* bytes, int32_t len, int64_t* code) {
  if (!ix || !code || (!bytes && len > 0) || len < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_seek: bad argument");
  if (column < 0 || (size_t)column >= ix->kw.size()) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_seek: keyword column out of range");
  const KeywordColumn& c = *ix->kw[(size_t)column];
  *code = keyword_seek_code(c.bytes.data(), c.off.data(), c.n_terms, bytes, len);
  return NRTGPU_OK;
}

int nrtgpu_index_keyword_range(const nrtgpu_index* ix, int32_t column, const uint8_t* lower, int32_t lower_len, const uint8_t* upper,
                               int32_t upper_len, int32_t flags, int64_t* lo, int64_t* hi) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_range: NULL index");
  if (column < 0 || (size_t)column >= ix->kw.size()) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_range: keyword column out of range");
  const KeywordColumn& c = *ix->kw[(size_t)column];
  return keyword_range_codes(c.bytes.data(), c.off.data(), c.n_terms, lower, lower_len, upper, upper_len, flags, lo, hi);
}

int nrtgpu_index_keyword_term(const nrtgpu_index* ix, int32_t column, int32_t ord, uint8_t* out, int32_t cap, int32_t* len) {
  if (!ix || !len) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_term: NULL argument");
  if (column < 0 || (size_t)column >= ix->kw.size()) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_term: keyword column out of range");
  const KeywordColumn& c = *ix->kw[(size_t)column];
  if (ord < 0 || ord >= c.n_terms) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_keyword_term: ordinal out of range");
  copy_term(c.bytes, c.off, ord, out, cap, len);
  return NRTGPU_OK;
}

int nrtgpu_index_set_live_docs(nrtgpu_index* ix, const uint8_t* live_docs) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_set_live_docs: NULL index");
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  NRT_CUDA_TRY(cudaDeviceSynchronize());   // searches in flight on this image finish against the old bitmap
  return upload_live_docs(ix, live_docs);
}

int nrtgpu_index_update_stats(nrtgpu_index* ix, const int64_t* term_df, const int64_t* field_doc_count, const int64_t* field_sum_ttf) {
  if (!ix || !field_doc_count || !field_sum_ttf) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_index_update_stats: NULL argument");
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  if (term_df) ix->term_df.assign(term_df, term_df + ix->n_terms);
  ix->field_doc_count.assign(field_doc_count, field_doc_count + ix->n_fields);
  ix->field_sum_ttf.assign(field_sum_ttf, field_sum_ttf + ix->n_fields);
  std::vector<float> caches((size_t)ix->n_fields * 256);
  for (int f = 0; f < ix->n_fields; ++f) {
    const int64_t dc = ix->field_doc_count[(size_t)f];
    const float avgdl = dc > 0 ? (float)((double)ix->field_sum_ttf[(size_t)f] / (double)dc) : 1.0f;
    bm25_cache(ix->field_k1[(size_t)f], ix->field_b[(size_t)f], avgdl, &caches[(size_t)f * 256]);
  }
  int rc;
  if ((rc = ix->caches.upload(caches.data(), caches.size()))) return rc;
  return compute_term_max_x(ix);   // the impacts are functions of the length cache
}

// ---- batch compilation (batch_plan.inc) + uploads ----
// compile the request and upload its clauses and queries into `b` (buffers are reused when large enough); asynchronous
// on `st`. What the compile-only entry points need (nrtgpu_score_docs, nrtgpu_rescore_query, nrtgpu_search_knn_filtered).
static int batch_compile(nrtgpu_batch* b, nrtgpu_index* ix, const BatchRequest& r, cudaStream_t st) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_prepare: NULL argument");
  int rc;
  if ((rc = compile_batch(ix->dict(), r, &b->cb))) return rc;
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  b->ix = ix; b->nq = r.nq; b->top_k = r.top_k;
  if ((rc = b->clauses.upload_async(b->cb.clauses.data(), b->cb.clauses.size(), st))) return rc;
  if (b->cb.tree) {
    if ((rc = b->nodes.upload_async(b->cb.nodes.data(), b->cb.nodes.size(), st))) return rc;
    if ((rc = b->node_begin.upload_async(b->cb.node_begin.data(), b->cb.node_begin.size(), st))) return rc;
    if ((rc = b->phrases.upload_async(b->cb.phrases.data(), b->cb.phrases.size(), st))) return rc;
    if ((rc = b->phrase_begin.upload_async(b->cb.phrase_begin.data(), b->cb.phrase_begin.size(), st))) return rc;
  }
  return b->queries.upload_async(b->cb.queries.data(), b->cb.queries.size(), st);
}

static int batch_filter_rows(nrtgpu_batch* b, const BatchRequest& r, cudaStream_t st);

// The multi-phrase unions of a compiled batch (union_kernel.cuh) into the batch's buffers, and every union clause's entry
// range into its uploaded clauses; asynchronous on `st`. The scratch is sized by the postings the unions gather
// (CompiledBatch::union_postings, capped by compile_tree) and the positions they merge.
static int union_build(nrtgpu_batch* b, nrtgpu_index* ix, cudaStream_t st) {
  const CompiledBatch& cb = b->cb;
  const int32_t n_alts = (int32_t)cb.union_term.size();
  std::vector<int64_t> gstart((size_t)n_alts + 1, 0), post((size_t)n_alts);
  std::vector<int32_t> au((size_t)n_alts), af((size_t)n_alts);
  for (int32_t u = 0; u < cb.n_unions(); ++u)
    for (int32_t a = cb.union_begin[(size_t)u]; a < cb.union_begin[(size_t)u + 1]; ++a) {
      const int32_t t = cb.union_term[(size_t)a];
      post[(size_t)a] = ix->term_off[(size_t)t];
      gstart[(size_t)a + 1] = gstart[(size_t)a] + (ix->term_off[(size_t)t + 1] - ix->term_off[(size_t)t]);
      au[(size_t)a] = u; af[(size_t)a] = ix->term_field[(size_t)t];
    }
  const int64_t S = gstart[(size_t)n_alts];
  int rc;
  if ((rc = b->u_alt_gstart.upload_async(gstart.data(), gstart.size(), st)) || (rc = b->u_alt_post.upload_async(post.data(), post.size(), st)) ||
      (rc = b->u_alt_term.upload_async(cb.union_term.data(), cb.union_term.size(), st)) ||
      (rc = b->u_alt_union.upload_async(au.data(), au.size(), st)) || (rc = b->u_alt_field.upload_async(af.data(), af.size(), st)) ||
      (rc = b->u_alt_weight.upload_async(cb.union_weight.data(), cb.union_weight.size(), st)) ||
      (rc = b->u_mode.upload_async(cb.union_scored.data(), cb.union_scored.size(), st)) ||
      (rc = b->u_clause.upload_async(cb.union_clause.data(), cb.union_clause.size(), st))) return rc;
  const size_t n1 = (size_t)std::max<int64_t>(S, 1);
  for (int i = 0; i < 2; ++i) if ((rc = b->u_keys[i].alloc(n1)) || (rc = b->u_vals[i].alloc(n1))) return rc;
  // (the entries of the batch's joins follow the union entries: join_build)
  if ((rc = b->u_head.alloc(n1)) || (rc = b->u_incl.alloc(n1)) || (rc = b->u_docs.alloc(n1 + cb.join_bound)) || (rc = b->u_first.alloc(n1)) ||
      (rc = b->u_score.alloc(n1 + cb.join_bound)) || (rc = b->u_npos.alloc(n1 + 1)) || (rc = b->u_pos_off.alloc(n1 + 1)) ||
      (rc = b->u_positions.alloc((size_t)std::max<int64_t>(cb.union_positions, 1)))) return rc;
  NRT_CUDA_TRY(cudaMemsetAsync(b->u_npos.p, 0, (n1 + 1) * sizeof(int32_t), st));
  UnionBuildLaunch U{};
  U.ix = ix->view(); U.n_alts = n_alts; U.alt_gstart = b->u_alt_gstart.p; U.alt_post = b->u_alt_post.p; U.alt_term = b->u_alt_term.p;
  U.alt_union = b->u_alt_union.p; U.alt_field = b->u_alt_field.p; U.alt_weight = b->u_alt_weight.p; U.union_mode = b->u_mode.p;
  U.n_gather = S; U.head = b->u_head.p; U.incl = b->u_incl.p; U.docs = b->u_docs.p; U.score = b->u_score.p; U.first = b->u_first.p;
  U.npos = b->u_npos.p; U.pos_off = b->u_pos_off.p; U.positions = b->u_positions.p;
  U.clauses = b->clauses.p; U.union_clause = b->u_clause.p; U.n_union_clauses = (int32_t)cb.union_clause.size();
  const unsigned grid = (unsigned)((S + 255) / 256);
  if (S > 0) {
    union_gather_kernel<<<grid, 256, 0, st>>>(U, b->u_keys[0].p, b->u_vals[0].p);
    NRT_CUDA_TRY(cudaGetLastError());
    int end_bit = 32;
    while (end_bit < 64 && (1ll << (end_bit - 32)) < (int64_t)cb.n_unions()) ++end_bit;
    cub::DoubleBuffer<uint64_t> keys(b->u_keys[0].p, b->u_keys[1].p);
    cub::DoubleBuffer<int32_t> vals(b->u_vals[0].p, b->u_vals[1].p);
    size_t tb = 0, ts = 0;
    NRT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, vals, (int)S, 0, end_bit, st));
    NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, ts, b->u_head.p, b->u_incl.p, thrust::plus<void>(), (int)S, st));
    size_t tp = 0;
    NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, tp, b->u_npos.p, b->u_pos_off.p + 1, thrust::plus<void>(), (int)S, st));
    if ((rc = b->u_temp.alloc(std::max(std::max(tb, ts), tp)))) return rc;
    tb = b->u_temp.bytes();
    NRT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(b->u_temp.p, tb, keys, vals, (int)S, 0, end_bit, st));
    U.keys = keys.Current(); U.vals = vals.Current();
    union_head_kernel<<<grid, 256, 0, st>>>(U);
    NRT_CUDA_TRY(cudaGetLastError());
    ts = b->u_temp.bytes();
    NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(b->u_temp.p, ts, b->u_head.p, b->u_incl.p, thrust::plus<void>(), (int)S, st));
    union_entry_kernel<<<grid, 256, 0, st>>>(U);
    NRT_CUDA_TRY(cudaGetLastError());
    if (cb.union_positions > 0) {
      tp = b->u_temp.bytes();
      // the exclusive scan of the position counts as pos_off[0] = 0 and the inclusive one behind it: both scans are the
      // int scan with thrust::plus that the library already instantiates (cub's InclusiveSum / ExclusiveSum kernels for
      // int spill 4 bytes on sm_90a)
      NRT_CUDA_TRY(cudaMemsetAsync(b->u_pos_off.p, 0, sizeof(int32_t), st));
      NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(b->u_temp.p, tp, b->u_npos.p, b->u_pos_off.p + 1, thrust::plus<void>(), (int)S, st));
      union_positions_kernel<<<grid, 256, 0, st>>>(U);
      NRT_CUDA_TRY(cudaGetLastError());
    }
  }
  if (U.n_union_clauses > 0) {
    union_patch_kernel<<<(unsigned)((U.n_union_clauses + 127) / 128), 128, 0, st>>>(U);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  b->u_view = UnionView{b->u_docs.p, b->u_score.p, b->u_pos_off.p, b->u_positions.p};
  b->u_gathered = S;
  return NRTGPU_OK;
}

// The block joins of a compiled batch (join_kernel.cuh) into the entry arrays behind its union entries (union_build ran
// first and sized them), and every join clause's entry range into its uploaded clauses; asynchronous on `st`. The child
// pass reads the image without its live docs and runs when the batch is built, without the search deadline. The scratch
// is sized by the joins' bounded child matches (CompiledBatch::join_bound, capped by compile_tree): the keys beyond the
// matches keep the sentinel ~0, which sorts after every real key, so the host never reads the match count back.
static int join_build(nrtgpu_batch* b, nrtgpu_index* ix, cudaStream_t st) {
  const CompiledBatch& cb = b->cb;
  const WorkPlan& p = b->plan;
  const int64_t n = cb.join_bound;
  const size_t n1 = (size_t)std::max<int64_t>(n, 1);
  const int64_t base = cb.n_unions() > 0 ? b->u_gathered : 0;
  int rc;
  if (cb.n_unions() == 0) {
    if ((rc = b->u_docs.alloc(n1)) || (rc = b->u_score.alloc(n1))) return rc;
    b->u_view = UnionView{b->u_docs.p, b->u_score.p, nullptr, nullptr};
  }
  if ((rc = b->j_work_query.upload_async(p.join_query.data(), p.join_query.size(), st)) ||
      (rc = b->j_work_slice.upload_async(p.join_slice.data(), p.join_slice.size(), st)) ||
      (rc = b->j_clause.upload_async(cb.join_clause.data(), cb.join_clause.size(), st)) ||
      (rc = b->j_mode.upload_async(cb.join_mode.data(), cb.join_mode.size(), st))) return rc;
  for (int i = 0; i < 2; ++i) if ((rc = b->j_keys[i].alloc(n1)) || (rc = b->j_scores[i].alloc(n1))) return rc;
  if ((rc = b->j_head.alloc(n1)) || (rc = b->j_incl.alloc(n1)) || (rc = b->j_count.alloc(1))) return rc;
  NRT_CUDA_TRY(cudaMemsetAsync(b->j_keys[0].p, 0xff, n1 * sizeof(uint64_t), st));
  NRT_CUDA_TRY(cudaMemsetAsync(b->j_count.p, 0, sizeof(unsigned int), st));
  if (!p.join_query.empty()) {   // the child pass
    BoolLaunchJ L{};
    L.ix = ix->view(); L.ix.live_bits = nullptr;
    L.clauses = b->clauses.p; L.queries = b->queries.p;
    L.work_query = b->j_work_query.p; L.work_slice = b->j_work_slice.p; L.n_work = (int32_t)p.join_query.size();
    L.n_slices = p.n_slices; L.top_k = b->top_k;
    L.nodes = b->nodes.p; L.node_begin = b->node_begin.p; L.phrases = b->phrases.p; L.phrase_begin = b->phrase_begin.p;
    L.aggs = nullptr;
    L.u = b->u_view;
    L.emit_keys = b->j_keys[0].p; L.emit_scores = b->j_scores[0].p; L.emit_count = b->j_count.p; L.emit_cap = n;
    L.join_q0 = cb.nq;
    bool_window_emit_kernel<<<(unsigned)L.n_work, kThreads, sizeof(BoolTreeSmemU), st>>>(L);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  JoinBuildLaunch J{};
  J.parent_bits = ix->parent_bits.p; J.n_words = (int32_t)((ix->n_docs + 31) / 32); J.n_joins = cb.n_joins(); J.n = n;
  J.head = b->j_head.p; J.incl = b->j_incl.p; J.mode = b->j_mode.p; J.base = base;
  J.docs = b->u_docs.p; J.score = b->u_score.p; J.clauses = b->clauses.p; J.join_clause = b->j_clause.p;
  J.keys = b->j_keys[0].p; J.scores = b->j_scores[0].p;
  if (n > 0) {
    int end_bit = 33;   // the join bits hold every join and the sentinel's all-ones above them
    while (end_bit < 64 && (1ll << (end_bit - 32)) <= (int64_t)cb.n_joins()) ++end_bit;
    cub::DoubleBuffer<uint64_t> keys(b->j_keys[0].p, b->j_keys[1].p);
    cub::DoubleBuffer<float> vals(b->j_scores[0].p, b->j_scores[1].p);
    size_t tb = 0, ts = 0;
    NRT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, vals, (int)n, 0, end_bit, st));
    NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, ts, b->j_head.p, b->j_incl.p, thrust::plus<void>(), (int)n, st));
    if ((rc = b->j_temp.alloc(std::max(tb, ts)))) return rc;
    tb = b->j_temp.bytes();
    NRT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(b->j_temp.p, tb, keys, vals, (int)n, 0, end_bit, st));
    J.keys = keys.Current(); J.scores = vals.Current();
    const unsigned grid = (unsigned)((n + 255) / 256);
    join_head_kernel<<<grid, 256, 0, st>>>(J);
    NRT_CUDA_TRY(cudaGetLastError());
    ts = b->j_temp.bytes();
    // (the int scan with thrust::plus that the library already instantiates: cub's InclusiveSum kernels for int spill)
    NRT_CUDA_TRY(cub::DeviceScan::InclusiveScan(b->j_temp.p, ts, b->j_head.p, b->j_incl.p, thrust::plus<void>(), (int)n, st));
    join_entry_kernel<<<grid, 256, 0, st>>>(J);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  join_patch_kernel<<<(unsigned)((cb.n_joins() + 127) / 128), 128, 0, st>>>(J);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// the KEYWORD after values of the queries with searchAfter: 0 (null) or a code 1 .. 2n + 1 of the column's n terms (n_distinct
// of the order's field on an image; the caller's n on a searcher)
static int check_keyword_after(const nrtgpu_sort_order* o, const int64_t* after, const nrtgpu_query* queries, int32_t nq,
                               const char* fn, const int32_t* n_terms = nullptr) {
  for (int j = 0; j < o->n_fields; ++j) {
    if (o->spec[j].kind != NRTGPU_SORT_KEYWORD) continue;
    const int64_t hi = 2 * (int64_t)(n_terms ? n_terms[j] : o->f[j].n_distinct) + 1;
    for (int q = 0; q < nq; ++q)
      if (queries[q].has_after) {
        const int64_t c = after[(size_t)q * o->n_fields + j];
        if (c < 0 || c > hi)
          NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": keyword after value " + std::to_string(c) + " of sort field " +
                                           std::to_string(j) + " is not a code of the column's " + std::to_string(hi / 2) + " terms");
      }
  }
  return NRTGPU_OK;
}

// a search batch: compile, plan the work list, upload, set up sorted searchAfter, allocate the results, launch
// slice_bounds_kernel and build the rows of the filter collectors
static int batch_build(nrtgpu_batch* b, nrtgpu_index* ix, const BatchRequest& r, cudaStream_t st) {
  int rc;
  if ((rc = batch_compile(b, ix, r, st))) return rc;
  const nrtgpu_sort* sort = r.sort;
  const nrtgpu_sort_order* sort_order = r.sort_order;
  const int32_t nq = r.nq, top_k = r.top_k;
  b->order = sort_order;
  b->ran = false; b->runs_recorded = 0;
  b->agg_shared = false;
  b->nest_kw_map.clear();
  if (sort_order) {   // fields-only order: the COLUMN key with the rank as its code; [score, ...]: kSortScoreRank
    b->sort_kind = sort_order->score_first ? kSortScoreRank : NRTGPU_SORT_COLUMN; b->sort_column = 0;
    b->sort_reverse = sort_order->score_first ? sort_order->score_reverse : 0; b->sort_missing_value = 0;
  } else {
    const bool sorted = b->cb.sorted;
    b->sort_kind = sorted ? sort->kind : 0; b->sort_column = sorted ? sort->column : 0; b->sort_reverse = sorted ? (sort->reverse != 0) : 0;
    b->sort_missing_value = sorted ? sort->missing_value : 0;
  }
  if (b->cb.n_unions() > 0 && (rc = union_build(b, ix, st))) return rc;
  WorkPlan& p = b->plan;
  plan_work(ix->dict(), ix->ctx->plan, b->cb, &p);
  if (b->cb.n_joins() > 0 && (rc = join_build(b, ix, st))) return rc;
  if ((rc = b->work_query.upload_async(p.work_query.data(), p.work_query.size(), st))) return rc;
  if ((rc = b->work_slice.upload_async(p.work_item.data(), p.work_item.size(), st))) return rc;
  if ((rc = b->known_hits.upload_async(p.known_hits.data(), p.known_hits.size(), st))) return rc;
  if ((rc = b->warm_exact.upload_async(p.warm_exact.data(), p.warm_exact.size(), st))) return rc;
  if (b->cb.sorted) {
    bool any_after = false;
    b->h_after_docs.assign((size_t)nq, 0);
    for (int qi = 0; qi < nq; ++qi) if (r.queries[qi].has_after) { any_after = true; b->h_after_docs[(size_t)qi] = r.queries[qi].after_doc; }
    if (sort_order) {
      // (the COLUMN key reads a missing code; ranks are never 0, so it is never used)
      if ((rc = b->sort_missing_code.alloc(1))) return rc;
      NRT_CUDA_TRY(cudaMemsetAsync(b->sort_missing_code.p, 0, sizeof(uint32_t), st));
      if ((rc = b->after_docs.upload_async(b->h_after_docs.data(), (size_t)nq, st))) return rc;
      const size_t nv = (size_t)nq * sort_order->n_fields;
      if (r.order_after && any_after)
        if ((rc = check_keyword_after(sort_order, r.order_after, r.queries, nq, "nrtgpu_search_sorted_fields"))) return rc;
      if (r.order_after) { if ((rc = b->after_values.upload_async(r.order_after, nv, st))) return rc; }
      else if ((rc = b->after_values.alloc(nv))) return rc;
      SortFieldsAfterLaunch A{};
      A.queries = b->queries.p; A.nq = nq; A.after_docs = b->after_docs.p; A.after_values = b->after_values.p;
      A.n_fields = sort_order->n_fields; A.score_first = sort_order->score_first ? 1 : 0; A.score_reverse = sort_order->score_reverse;
      A.n_rank = sort_order->n_rank;
      for (int i = 0; i < sort_order->n_rank; ++i) A.f[i] = sort_order->f[i + A.score_first];
      A.perm = sort_order->perm.p; A.n_docs = ix->n_docs; A.doc_base = ix->doc_base;
      if (any_after) sort_fields_after_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, st>>>(A);
      NRT_CUDA_TRY(cudaGetLastError());
      if ((rc = b->out_sort_values.alloc(nv * top_k))) return rc;
    } else {
      if ((rc = b->sort_missing_code.alloc(1))) return rc;
      if ((rc = b->after_docs.upload_async(b->h_after_docs.data(), (size_t)nq, st))) return rc;
      if (sort->after_values) { if ((rc = b->after_values.upload_async(sort->after_values, (size_t)nq, st))) return rc; }
      else if ((rc = b->after_values.alloc((size_t)nq))) return rc;
      SortAfterLaunch A;
      A.queries = b->queries.p; A.nq = nq; A.after_docs = b->after_docs.p; A.after_values = b->after_values.p;
      A.kind = sort->kind; A.reverse = sort->reverse != 0; A.doc_base = ix->doc_base; A.n_docs = ix->n_docs;
      const bool col = sort->kind == NRTGPU_SORT_COLUMN;
      A.distinct = col ? ix->col_distinct[(size_t)sort->column]->p : nullptr;
      A.n_distinct = col ? ix->col_n_distinct[(size_t)sort->column] : 0;
      A.missing_value = sort->missing_value; A.missing_code = b->sort_missing_code.p;
      sort_after_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, st>>>(A);
      NRT_CUDA_TRY(cudaGetLastError());
      if ((rc = b->out_sort_values.alloc((size_t)nq * top_k))) return rc;
    }
  }
  if ((rc = b->theta.alloc((size_t)nq))) return rc;
  if ((rc = b->total_hits.alloc((size_t)nq))) return rc;
  if ((rc = b->slice_keys.alloc((size_t)nq * p.n_lists * top_k))) return rc;
  if ((rc = b->slice_cnt.alloc((size_t)nq * p.n_lists))) return rc;
  if ((rc = b->out_docs.alloc((size_t)nq * top_k))) return rc;
  if ((rc = b->out_scores.alloc((size_t)nq * top_k))) return rc;
  if ((rc = b->out_counts.alloc((size_t)nq))) return rc;
  if ((rc = b->pruned.alloc((size_t)nq))) return rc;
  if ((rc = b->terminated.alloc((size_t)nq))) return rc;
  if (p.n_probe_simple + p.n_probe_generic > 0) {
    // the state of every query that no work item changes, which each item copies instead of deriving it ...
    if ((rc = b->pquery.alloc((size_t)nq))) return rc;
    v3::ProbeQueryLaunch Q;
    Q.ix = ix->view(); Q.clauses = b->clauses.p; Q.queries = b->queries.p; Q.field_min_norm = ix->field_min_norm.p;
    Q.warm_exact = b->warm_exact.p; Q.n_gran = p.n_gran; Q.out = b->pquery.p;
    v3::probe_query_kernel<<<(unsigned)nq, v3::kUbt, 0, st>>>(Q);
    NRT_CUDA_TRY(cudaGetLastError());
    // ... and the posting offsets of every (query, term slot) at the part boundaries only (skip data for the long lists,
    // one lower_bound for the short ones) and at the end of an exact warm-up (the records' warm_gran); the granule offsets
    // inside a slice are read from gran_tab by the kernel
    const int64_t total = (int64_t)nq * v3::kT * v3::boundary_entries(p.n_slices, p.parts_max);
    if ((rc = b->sbounds.alloc((size_t)total))) return rc;
    if ((rc = b->work_counter.alloc(2))) return rc;
    v3::SliceBoundsLaunch S;
    S.ix = Q.ix; S.clauses = b->clauses.p; S.queries = b->queries.p; S.pquery = b->pquery.p; S.nq = nq; S.n_slices = p.n_slices;
    S.slice_gran = p.slice_docs / v3::kGran; S.n_gran = p.n_gran; S.parts_max = p.parts_max; S.sbounds = b->sbounds.p;
    v3::slice_bounds_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  if (!b->ev[0][0]) for (auto& r : b->ev) for (auto& e : r) NRT_CUDA_TRY(cudaEventCreate(&e));
  return batch_filter_rows(b, r, st);
}

int nrtgpu_batch_prepare(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                         int32_t total_hits_threshold, int32_t flags, nrtgpu_batch** out) {
  if (!out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_prepare: NULL argument");
  std::unique_ptr<nrtgpu_batch> b(new nrtgpu_batch);
  int rc = batch_build(b.get(), ix, BatchRequest{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags}, (cudaStream_t)0);
  if (rc) return rc;
  NRT_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)0));
  *out = b.release();
  return NRTGPU_OK;
}

static BatchRequest tree_request(const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                                 const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags);
static int phrase_request(BatchRequest* r, const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms,
                          int32_t n_phrase_terms);

int nrtgpu_batch_prepare_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                              int32_t n_nodes, const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                              int32_t total_hits_threshold, int32_t flags, nrtgpu_batch** out) {
  if (!out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_prepare: NULL argument");
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  std::unique_ptr<nrtgpu_batch> b(new nrtgpu_batch);
  int rc = batch_build(b.get(), ix, tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, total_hits_threshold, flags),
                       (cudaStream_t)0);
  if (rc) return rc;
  NRT_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)0));
  *out = b.release();
  return NRTGPU_OK;
}

int nrtgpu_batch_prepare_tree_phrases(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                                      int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                      const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                                      int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags, nrtgpu_batch** out) {
  if (!out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_prepare: NULL argument");
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  BatchRequest r = tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, total_hits_threshold, flags);
  int rc = phrase_request(&r, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc) return rc;
  r.unions = true;
  std::unique_ptr<nrtgpu_batch> b(new nrtgpu_batch);
  if ((rc = batch_build(b.get(), ix, r, (cudaStream_t)0))) return rc;
  NRT_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)0));
  *out = b.release();
  return NRTGPU_OK;
}

// the probe kernel's parameters for the batch's own outputs (no collectors, no stats; the work items are set at launch)
static v3::ProbeLaunch probe_params(nrtgpu_batch* b) {
  v3::ProbeLaunch P;
  P.ix = b->ix->view(); P.pquery = b->pquery.p; P.sbounds = b->sbounds.p;
  P.stats = nullptr;
  P.known_hits = b->ix->live_bits.p ? nullptr : b->known_hits.p;   // (deletes installed after the batch was prepared: list lengths no longer bound the hits)
#ifdef NRT_PROBE_KNOCK
  { const char* e = getenv("NRTGPU_KNOCK"); P.knock = e ? atoi(e) : 0; }   // profiling builds only (tools/knock.py)
#else
  P.knock = 0;
#endif
  P.n_lists = b->plan.n_lists; P.parts_max = b->plan.parts_max; P.n_slices = b->plan.n_slices; P.top_k = b->top_k; P.slice_docs = b->plan.slice_docs; P.n_gran = b->plan.n_gran;
  P.threshold = b->cb.threshold; P.pruned = b->pruned.p; P.theta = b->theta.p; P.total_hits = b->total_hits.p;
  P.slice_keys = b->slice_keys.p; P.slice_cnt = b->slice_cnt.p;
  P.deadline_ns = b->limits_active ? b->deadline_ns : 0; P.clock0 = b->clock0.p; P.timed_out = b->timed_out.p;
  P.terminate_after = b->ta_scalar; P.terminated = b->terminated.p;
  P.sort_kind = b->sort_kind; P.sort_reverse = b->sort_reverse;
  P.sort_codes = b->order ? b->order->rank.p : b->sort_kind == NRTGPU_SORT_COLUMN ? b->ix->col_code[(size_t)b->sort_column]->p : nullptr;
  P.sort_missing_code = b->sort_missing_code.p;
  P.aggs = nullptr;
  return P;
}

// the probe kernel over the batch's work items: the simple ones, then the generic ones (queue heads work_counter[0], [1])
// multi: the collectors count a SORTED_SET keyword column, so the generic items run the kMulti instantiation (without the
// profiling counters)
static int probe_launch(nrtgpu_batch* b, v3::ProbeLaunch P, bool debug, bool multi, cudaStream_t st) {
  // configuration A (3 CTAs / SM) for the pruned sweeps of TOP_SCORES, B (4 CTAs / SM) where every posting is visited
  const bool cfg_b_simple = ix_ctx_probe_cfg(b->ix->ctx, P.threshold >= (int64_t)INT32_MAX);
  const bool cfg_b_generic = ix_ctx_probe_cfg(b->ix->ctx, true);
  auto launch = [&](auto simple_tag, bool cfg_b, int n_items) {
    constexpr bool S = decltype(simple_tag)::value;
    if (!S && multi) {
      const int ctas = cfg_b ? v3::kCtasB : v3::kCtasA;
      const int grid = std::min(ctas * b->ix->ctx->plan.sm_count, n_items);
      if (cfg_b) v3::posting_probe_kernel<false, false, v3::kCtasB, v3::kStageB, true><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageB>), st>>>(P);
      else v3::posting_probe_kernel<false, false, v3::kCtasA, v3::kStageA, true><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageA>), st>>>(P);
    } else if (cfg_b) {
      const int grid = std::min(v3::kCtasB * b->ix->ctx->plan.sm_count, n_items);
      if (debug) v3::posting_probe_kernel<S, true, v3::kCtasB, v3::kStageB><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageB>), st>>>(P);
      else v3::posting_probe_kernel<S, false, v3::kCtasB, v3::kStageB><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageB>), st>>>(P);
    } else {
      const int grid = std::min(v3::kCtasA * b->ix->ctx->plan.sm_count, n_items);
      if (debug) v3::posting_probe_kernel<S, true, v3::kCtasA, v3::kStageA><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageA>), st>>>(P);
      else v3::posting_probe_kernel<S, false, v3::kCtasA, v3::kStageA><<<grid, v3::kThreads, sizeof(v3::ProbeSmemT<v3::kStageA>), st>>>(P);
    }
  };
  if (b->plan.n_probe_simple > 0) {
    P.work_query = b->work_query.p; P.work_slice = b->work_slice.p; P.n_work = b->plan.n_probe_simple; P.work_counter = b->work_counter.p;
    P.stats = debug ? b->probe_stats.p : nullptr;
    launch(std::true_type{}, cfg_b_simple, b->plan.n_probe_simple);
  }
  if (b->plan.n_probe_generic > 0) {
    P.work_query = b->work_query.p + b->plan.n_probe_simple; P.work_slice = b->work_slice.p + b->plan.n_probe_simple;
    P.n_work = b->plan.n_probe_generic; P.work_counter = b->work_counter.p + 1;
    P.stats = debug ? b->probe_stats.p + v3::kProbeStats : nullptr;
    launch(std::false_type{}, cfg_b_generic, b->plan.n_probe_generic);
  }
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// The batch's engine over its work items: the probe kernel, or bool_window_kernel for wide and tree batches, with the
// additional collectors `aggs` (device pointer, NULL: none). Pass 1 (p2_total NULL) counts into the batch's own totalHits and
// flags under its limits. The top-hits run of batch_nested_top_hits counts totalHits into p2_total and the probe kernel's
// pruned / terminated into p2_flags [2 * nq], without deadline or terminateAfter; the caller has reset the engine's theta,
// slice counts and queue heads. multi: a collector counts a SORTED_SET keyword column (the kMulti instantiations).
static int batch_engine_launch(nrtgpu_batch* b, const AggLaunch* aggs, bool multi, unsigned long long* p2_total, int32_t* p2_flags,
                               bool debug, cudaStream_t st) {
  const bool p2 = p2_total != nullptr;
  if (!b->cb.wide) {
    v3::ProbeLaunch P = probe_params(b);
    P.aggs = aggs;
    if (p2) { P.total_hits = p2_total; P.pruned = p2_flags; P.terminated = p2_flags + b->nq; P.deadline_ns = 0; P.terminate_after = 0; }
    return probe_launch(b, P, debug && !p2, multi, st);
  }
  BoolLaunch L;
  L.ix = b->ix->view();
  L.nodes = nullptr; L.node_begin = nullptr; L.phrases = nullptr; L.phrase_begin = nullptr;
  L.clauses = b->clauses.p; L.queries = b->queries.p;
  L.work_query = b->work_query.p; L.work_slice = b->work_slice.p;
  L.n_work = b->plan.n_work(); L.n_slices = b->plan.n_lists; L.top_k = b->top_k;
  L.theta = b->theta.p; L.total_hits = p2 ? p2_total : b->total_hits.p;
  L.slice_keys = b->slice_keys.p; L.slice_cnt = b->slice_cnt.p;
  L.deadline_ns = (!p2 && b->limits_active) ? b->deadline_ns : 0; L.clock0 = b->clock0.p; L.timed_out = b->timed_out.p;
  L.aggs = aggs;
  const unsigned grid = (unsigned)b->plan.n_work();
  if (b->cb.tree && (b->cb.n_unions() > 0 || b->cb.n_joins() > 0)) {   // union or join slots
    BoolLaunchU LU;
    static_cast<BoolLaunch&>(LU) = L;
    LU.nodes = b->nodes.p; LU.node_begin = b->node_begin.p; LU.phrases = b->phrases.p; LU.phrase_begin = b->phrase_begin.p;
    LU.u = b->u_view;
    if (multi) bool_window_union_kernel<true, true><<<grid, kThreads, sizeof(BoolTreeSmemU), st>>>(LU);
    else if (aggs) bool_window_union_kernel<true><<<grid, kThreads, sizeof(BoolTreeSmemU), st>>>(LU);
    else bool_window_union_kernel<false><<<grid, kThreads, sizeof(BoolTreeSmemU), st>>>(LU);
  } else if (b->cb.tree) {
    L.nodes = b->nodes.p; L.node_begin = b->node_begin.p; L.phrases = b->phrases.p; L.phrase_begin = b->phrase_begin.p;
    if (multi) bool_window_kernel<true, true, true><<<grid, kThreads, sizeof(BoolTreeSmem), st>>>(L);
    else if (aggs) bool_window_kernel<true, true><<<grid, kThreads, sizeof(BoolTreeSmem), st>>>(L);
    else bool_window_kernel<true, false><<<grid, kThreads, sizeof(BoolTreeSmem), st>>>(L);
  } else {
    if (multi) bool_window_kernel<false, true, true><<<grid, kThreads, sizeof(BoolSmem), st>>>(L);
    else if (aggs) bool_window_kernel<false, true><<<grid, kThreads, sizeof(BoolSmem), st>>>(L);
    else bool_window_kernel<false, false><<<grid, kThreads, sizeof(BoolSmem), st>>>(L);
  }
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// a column's bucket codes and sorted distinct values in an image (NULL in an image without docs: it has no such arrays)
static const uint32_t* ix_col_code(const nrtgpu_index* ix, int32_t c) {
  return (size_t)c < ix->col_code.size() ? ix->col_code[(size_t)c]->p : nullptr;
}
static const uint64_t* ix_col_distinct(const nrtgpu_index* ix, int32_t c) {
  return (size_t)c < ix->col_distinct.size() ? ix->col_distinct[(size_t)c]->p : nullptr;
}

// Allocates the tables of the batch's collectors in its own buffers, n_buckets[i] buckets for terms aggregation i (1 for a
// filter aggregation), and
// resets them on `st`: counts to 0, min words to +inf and max words to -inf in ordered-double space, sums to 0.0 (the
// "unset" values are applied at fetch). Fills every field of *t but the codes and distinct values, which are the caller's.
static int batch_agg_tables(nrtgpu_batch* b, const int32_t* n_buckets, cudaStream_t st, AggTables* t) {
  int rc;
  for (size_t i = 0; i < b->cb.aggs.size(); ++i) {
    const nrtgpu_aggregation& a = b->cb.aggs[i];
    if (a.kind == NRTGPU_AGG_TERMS || a.kind == NRTGPU_AGG_FILTER) {
      t->n_buckets[i] = n_buckets[i];
      if ((rc = b->agg_counts[i].alloc((size_t)b->nq * (size_t)std::max(n_buckets[i], 1)))) return rc;
      NRT_CUDA_TRY(cudaMemsetAsync(b->agg_counts[i].p, 0, b->agg_counts[i].bytes(), st));
      t->counts[i] = b->agg_counts[i].p;
    } else {
      if ((rc = b->agg_dvals[i].alloc((size_t)b->nq))) return rc;
      NRT_CUDA_TRY(cudaMemsetAsync(b->agg_dvals[i].p, a.kind == NRTGPU_AGG_MIN ? 0xff : 0x00, b->agg_dvals[i].bytes(), st));
      t->dvals[i] = b->agg_dvals[i].p;
    }
  }
  for (size_t j = 0; j < b->cb.nested.size(); ++j) {   // nested min / max / sum: one word per (query, parent bucket), as above
    const nrtgpu_nested_aggregation& n = b->cb.nested[j];
    if (n.kind == NRTGPU_AGG_TOP_HITS) continue;
    const int32_t nb = n_buckets[n.parent];
    if ((rc = b->nest_words[j].alloc((size_t)b->nq * (size_t)std::max(nb, 1)))) return rc;
    NRT_CUDA_TRY(cudaMemsetAsync(b->nest_words[j].p, n.kind == NRTGPU_AGG_MIN ? 0xff : 0x00, b->nest_words[j].bytes(), st));
    t->nest_words[j] = b->nest_words[j].p;
  }
  return NRTGPU_OK;
}

// The codes every aggregation of the run counts through (agg_codes): its column's codes in agg_tab, or, for an aggregation
// a row gates (batch_filter_rows), agg_row_codes_kernel's: a filter collector is a one-bucket terms aggregation to the
// probe kernel, and a terms aggregation under a filter counts its column's codes where the filter's row passes. So the
// probe kernel's collector is the one it was before filter collectors, and the launches without them run the same code.
static int batch_agg_codes(nrtgpu_batch* b, cudaStream_t st) {
  for (size_t i = 0; i < b->cb.aggs.size(); ++i) {
    b->agg_codes[i] = b->agg_tab.codes[i];
    const uint32_t* row = b->agg_gate[i];
    if (!row) continue;
    const int32_t n = b->ix->n_docs;
    if (const int64_t* off = b->agg_tab.offsets[i]) {   // SORTED_SET keyword terms: every value of a passing doc
      if (int rc = b->agg_fcodes[i].alloc((size_t)std::max<int64_t>(b->ix->kw[(size_t)b->cb.aggs[i].column]->n_values, 1))) return rc;
      agg_row_value_codes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(row, b->agg_tab.codes[i], off, n, b->agg_fcodes[i].p);
    } else {
      if (int rc = b->agg_fcodes[i].alloc((size_t)n)) return rc;
      agg_row_codes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(row, b->cb.aggs[i].kind == NRTGPU_AGG_FILTER ? nullptr : b->agg_tab.codes[i],
                                                                      n, b->agg_fcodes[i].p);
    }
    NRT_CUDA_TRY(cudaGetLastError());
    b->agg_codes[i] = b->agg_fcodes[i].p;
  }
  return NRTGPU_OK;
}

int nrtgpu_batch_run(nrtgpu_batch* b, void* stream_) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_run: NULL batch");
  cudaStream_t st = (cudaStream_t)stream_;
  int rc_dbg = 0;
  NRT_CUDA_TRY(cudaSetDevice(b->ix->ctx->device));
  NRT_CUDA_TRY(cudaMemsetAsync(b->theta.p, 0, b->theta.bytes(), st));
  NRT_CUDA_TRY(cudaMemsetAsync(b->total_hits.p, 0, b->total_hits.bytes(), st));
  NRT_CUDA_TRY(cudaMemsetAsync(b->slice_cnt.p, 0, b->slice_cnt.bytes(), st));
  NRT_CUDA_TRY(cudaMemsetAsync(b->pruned.p, 0, b->pruned.bytes(), st));
  NRT_CUDA_TRY(cudaMemsetAsync(b->terminated.p, 0, b->terminated.bytes(), st));
  if (b->work_counter.p) NRT_CUDA_TRY(cudaMemsetAsync(b->work_counter.p, 0, b->work_counter.bytes(), st));
  if (b->limits_active) {   // every engine, and batches without work items: batch_fetch_impl reads timed_out of THIS run
    NRT_CUDA_TRY(cudaMemsetAsync(b->clock0.p, 0, sizeof(unsigned long long), st));
    NRT_CUDA_TRY(cudaMemsetAsync(b->timed_out.p, 0, b->timed_out.bytes(), st));
  }
  // aggregation outputs start unset on every run, work items or not: batch_fetch_aggs reads those of THIS run (a searcher
  // resets its shared tables once per call, before the first leaf runs)
  if (!b->agg_shared && !b->cb.aggs.empty()) {
    AggTables& t = b->agg_tab;
    t = AggTables{};
    int32_t nb[kMaxAggs] = {};
    for (size_t i = 0; i < b->cb.aggs.size(); ++i) {
      const int32_t c = b->cb.aggs[i].column;
      nb[i] = 1;   // (a filter's one bucket)
      if (b->cb.aggs[i].kind != NRTGPU_AGG_TERMS) continue;
      if (agg_keyword(b->cb.aggs[i])) {   // ordinals of the image's dictionary
        const KeywordColumn& k = *b->ix->kw[(size_t)c];
        nb[i] = k.n_terms; t.codes[i] = k.codes.p; t.offsets[i] = k.doc_off.p;
        continue;
      }
      nb[i] = b->ix->col_n_distinct[(size_t)c];
      t.codes[i] = ix_col_code(b->ix, c); t.distinct[i] = ix_col_distinct(b->ix, c);
    }
    if ((rc_dbg = batch_agg_tables(b, nb, st, &t))) return rc_dbg;
  }
  const bool debug = b->ix->ctx->debug_modes;
  cudaEvent_t* ev = b->ev[b->runs_recorded % nrtgpu_batch::kEvRing];
  NRT_CUDA_TRY(cudaEventRecord(ev[0], st));
  if (b->plan.n_work() > 0) {
    const AggLaunch* aggs = nullptr;
    bool multi = false;   // a SORTED_SET keyword terms aggregation
    if (!b->cb.aggs.empty()) {   // pass 1 of the collectors, on either engine
      const AggTables& t = b->agg_tab;
      if ((rc_dbg = batch_agg_codes(b, st))) return rc_dbg;
      AggLaunch A; std::memset(&A, 0, sizeof(A));
      A.n_aggs = (int32_t)b->cb.aggs.size();
      for (int i = 0; i < A.n_aggs; ++i) {
        const nrtgpu_aggregation& a = b->cb.aggs[(size_t)i];
        A.a[i].kind = a.kind; A.a[i].column = a.column; A.a[i].value_type = a.value_type;
        if (a.kind == NRTGPU_AGG_FILTER) {   // a one-bucket terms aggregation over the image's column without a has array
          A.a[i].kind = NRTGPU_AGG_TERMS; A.a[i].column = b->ix->n_columns;
        }
        if (agg_keyword(a)) { A.a[i].column = b->ix->n_columns; A.offsets[i] = t.offsets[i]; }   // (codes alone say which docs have a term)
        if (a.kind == NRTGPU_AGG_TERMS || a.kind == NRTGPU_AGG_FILTER) {
          A.a[i].n_buckets = t.n_buckets[i];
          A.a[i].counts = t.counts[i]; A.codes[i] = b->agg_codes[i];
        } else {
          A.a[i].dvals = t.dvals[i];
        }
        A.nested_begin[i + 1] = A.nested_begin[i];   // pass 1: the nested min / max / sum collectors
        for (size_t j = 0; j < b->cb.nested.size(); ++j) {
          const nrtgpu_nested_aggregation& n = b->cb.nested[j];
          if (n.parent != i || n.kind == NRTGPU_AGG_TOP_HITS) continue;
          AggNestedDev& d = A.nested[A.nested_begin[i + 1]++];
          d.kind = n.kind; d.column = n.column; d.value_type = n.value_type; d.dvals = t.nest_words[j];
        }
        multi |= A.offsets[i] != nullptr;
      }
      if ((rc_dbg = b->agg_launch.upload_async(&A, 1, st))) return rc_dbg;
      NRT_CUDA_TRY(cudaStreamSynchronize(st));   // A is a stack object
      aggs = b->agg_launch.p;
    }
    if (debug && !b->cb.wide) {
      if (!b->probe_stats.p && (rc_dbg = b->probe_stats.alloc(2 * v3::kProbeStats))) return rc_dbg;
      NRT_CUDA_TRY(cudaMemsetAsync(b->probe_stats.p, 0, 2 * v3::kProbeStats * sizeof(unsigned long long), st));
    }
    if ((rc_dbg = batch_engine_launch(b, aggs, multi, nullptr, nullptr, debug, st))) return rc_dbg;
  }
  NRT_CUDA_TRY(cudaEventRecord(ev[1], st));
  if (debug && b->probe_stats.p && !b->cb.wide) {
    unsigned long long h[2 * v3::kProbeStats];
    NRT_CUDA_TRY(cudaMemcpyAsync(h, b->probe_stats.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    NRT_CUDA_TRY(cudaStreamSynchronize(st));
    for (int k = 0; k < 2; ++k) {
      const unsigned long long* x = h + v3::kProbeStats * k;
      if (x[0]) fprintf(stderr, "[nrtgpu probe %s] longest item %llu cyc; CTA busy: mean %.0f max %llu cyc; warm-up items %llu, %.0f cyc each; per item: flush %.0f cyc (%.0f in flush_top_k), TMA wait %.0f cyc\n", k == 0 ? "simple" : "generic",
                        x[8], (double)x[9] / std::min<double>((double)x[0], (double)(v3::kCtasA * b->ix->ctx->plan.sm_count)), x[10], x[11], x[11] ? (double)x[12] / x[11] : 0.0, (double)x[13] / x[0], (double)x[15] / x[0], (double)x[14] / x[0]);
      if (x[0]) fprintf(stderr, "[nrtgpu probe %s] %llu items, %.0f cyc/item (set-up %.0f), %.2f runs/item (%.2f staged), %.1f rounds/item, %llu driver postings (%.0f/item), %.0f queued/item, %.0f keys admitted/item, %.2f flushes/item\n",
                        k == 0 ? "simple" : "generic", x[0], (double)x[1] / x[0], (double)x[6] / x[0], (double)x[2] / x[0], (double)x[5] / x[0],
                        (double)x[7] / x[0], x[3], (double)x[3] / x[0], (double)x[16] / x[0], (double)x[17] / x[0], (double)x[4] / x[0]);
      if (k == 0 && x[0]) fprintf(stderr, "[nrtgpu probe simple] roles: %llu items start without a threshold (%.1f%% of item cycles; slice 0 %llu, slice 1 %llu); "
                                  "%llu items end with stale roles (%.1f%% of item cycles, %.0f cyc each, %llu driver postings, %llu in lists that turned non-essential; slice 0 %llu, slice 1 %llu)\n",
                                  x[18], 100.0 * (double)x[19] / (double)x[1], x[20], x[21], x[22], 100.0 * (double)x[23] / (double)x[1],
                                  x[22] ? (double)x[23] / x[22] : 0.0, x[24], x[25], x[26], x[27]);
      if (k == 0 && x[28]) fprintf(stderr, "[nrtgpu probe simple] exact warm-ups: %llu items, %llu driver postings, %.0f cyc each\n",
                                   x[28], x[29], (double)x[30] / x[28]);
    }
  }
  MergeLaunch M;
  M.slice_keys = b->slice_keys.p; M.slice_cnt = b->slice_cnt.p;
  M.n_lists = b->plan.n_lists; M.top_k = b->top_k; M.nq = b->nq; M.doc_base = b->ix->doc_base;
  M.out_docs = b->o_docs(); M.out_scores = b->o_scores(); M.out_counts = b->o_counts();
  M.total_hits = b->total_hits.p; M.pruned = b->pruned.p; M.terminated = b->terminated.p; M.terminate_after = b->ta_scalar;
  M.out_total = b->bound_total; M.out_flags = b->bound_flags;
  M.theta = !b->cb.wide ? b->theta.p : nullptr;
  M.known_hits = (!b->cb.wide && !b->ix->live_bits.p) ? b->known_hits.p : nullptr;
  merge_slices_kernel<<<b->nq, kMergeThreads, 0, st>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  if (b->order) {   // FieldDoc values of every field; score-first orders map ranks back to docs
    const nrtgpu_sort_order* o = b->order;
    SortFieldsValuesLaunch V{};
    V.docs = b->o_docs(); V.counts = b->o_counts(); V.nq = b->nq; V.top_k = b->top_k; V.doc_base = b->ix->doc_base;
    V.n_fields = o->n_fields; V.score_first = o->score_first ? 1 : 0; V.score_reverse = o->score_reverse;
    for (int i = 0; i < o->n_fields; ++i) V.f[i] = o->f[i];
    V.perm = o->perm.p; V.scores = b->o_scores(); V.out_values = b->o_sort_values();
    const int n = b->nq * b->top_k;
    sort_fields_values_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(V);
    NRT_CUDA_TRY(cudaGetLastError());
  } else if (b->sort_kind != NRTGPU_SORT_RELEVANCE) {   // FieldDoc values of the final hits; scores become NaN
    SortValuesLaunch V;
    V.docs = b->o_docs(); V.counts = b->o_counts(); V.nq = b->nq; V.top_k = b->top_k; V.doc_base = b->ix->doc_base; V.kind = b->sort_kind;
    const bool col = b->sort_kind == NRTGPU_SORT_COLUMN;
    V.c64 = col ? b->ix->col64[(size_t)b->sort_column]->p : nullptr; V.c32 = col ? b->ix->col32[(size_t)b->sort_column]->p : nullptr;
    V.has = col ? b->ix->col_has[(size_t)b->sort_column]->p : nullptr; V.missing_value = b->sort_missing_value;
    V.out_values = b->o_sort_values(); V.out_scores = b->o_scores();
    const int n = b->nq * b->top_k;
    sort_values_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(V);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  NRT_CUDA_TRY(cudaEventRecord(ev[2], st));
  b->runs_recorded++;
  b->ran = true;
  return NRTGPU_OK;
}

static int batch_fetch_impl(nrtgpu_batch* b, void* stream_, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                            int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  if (!b || !b->ran) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_fetch: batch has not run");
  cudaStream_t st = (cudaStream_t)stream_;
  size_t n = (size_t)b->nq * b->top_k;
  if (out_docs) NRT_CUDA_TRY(cudaMemcpyAsync(out_docs, b->o_docs(), n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (out_scores) NRT_CUDA_TRY(cudaMemcpyAsync(out_scores, b->o_scores(), n * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (out_counts) NRT_CUDA_TRY(cudaMemcpyAsync(out_counts, b->o_counts(), (size_t)b->nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (out_total_hits) NRT_CUDA_TRY(cudaMemcpyAsync(out_total_hits, b->total_hits.p, (size_t)b->nq * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  std::vector<int32_t>& pr = b->h_flags;
  pr.resize(3 * (size_t)b->nq);
  NRT_CUDA_TRY(cudaMemcpyAsync(pr.data(), b->pruned.p, (size_t)b->nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(pr.data() + b->nq, b->terminated.p, (size_t)b->nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  const bool has_to = b->timed_out.p != nullptr && b->limits_active;
  if (has_to) NRT_CUDA_TRY(cudaMemcpyAsync(pr.data() + 2 * (size_t)b->nq, b->timed_out.p, (size_t)b->nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  bool any_timeout = false;
  for (int i = 0; i < b->nq; ++i) {
    const bool term = pr[(size_t)b->nq + i] != 0;
    const bool to = has_to && pr[2 * (size_t)b->nq + i] != 0;
    any_timeout |= to;
    // TerminateAfterWrapper.java:85-90: an early-terminated search reports (hits counted, GREATER_THAN_OR_EQUAL_TO)
    if (out_relation) out_relation[i] = (pr[(size_t)i] || term || to) ? 1 : 0;
    if (out_terminated_early) out_terminated_early[i] = term ? 1 : 0;
    if (out_hit_timeout) out_hit_timeout[i] = to ? 1 : 0;
    if (out_total_hits && pr[(size_t)i] && !term && !to && !b->ix->live_bits.p && (size_t)i < b->plan.known_hits.size() && (int64_t)b->plan.known_hits[(size_t)i] > out_total_hits[i])
      out_total_hits[i] = (int64_t)b->plan.known_hits[(size_t)i];   // pruned search: the count is a lower bound; so is the longest list
    if (term && out_total_hits && b->terminate_after_max_recall > 0 && out_total_hits[i] > b->terminate_after_max_recall)
      out_total_hits[i] = b->terminate_after_max_recall;
  }
  // SearchCutoffWrapper.java:164-174: with noPartialResults a timeout is an error (CollectionTimeoutException), else the
  // partial results are returned and hitTimeout is set
  if (any_timeout && b->disallow_partial) NRT_FAIL(NRTGPU_ERR_TIMEOUT, "Search collection exceeded timeout of " + std::to_string(b->timeout_sec) + "s");
  return NRTGPU_OK;
}

int nrtgpu_batch_fetch(nrtgpu_batch* b, void* stream_, int32_t* out_docs, float* out_scores,
                       int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation) {
  return batch_fetch_impl(b, stream_, out_docs, out_scores, out_counts, out_total_hits, out_relation, nullptr, nullptr);
}

int nrtgpu_batch_fetch_ex(nrtgpu_batch* b, void* stream_, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                          int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  return batch_fetch_impl(b, stream_, out_docs, out_scores, out_counts, out_total_hits, out_relation, out_hit_timeout, out_terminated_early);
}

// The FieldDoc values of sorted nested top hits under order o (sort_fields_values_kernel): n lists of top_k docs that hold
// rank + doc_base become global docs, their scores (key score words) NaN, and values [n][top_k][n_fields] are written; 0
// past counts
static int sorted_hit_values(const nrtgpu_sort_order* o, int32_t doc_base, int32_t* docs, const int32_t* counts, float* scores, int n,
                             int top_k, int64_t* values, cudaStream_t st) {
  SortFieldsValuesLaunch V{};
  V.docs = docs; V.counts = counts; V.nq = n; V.top_k = top_k; V.doc_base = doc_base; V.n_fields = o->n_fields;
  V.score_first = o->score_first ? 1 : 0; V.score_reverse = o->score_reverse; V.ranks = 1;
  for (int i = 0; i < o->n_fields; ++i) V.f[i] = o->f[i];
  V.perm = o->perm.p; V.scores = scores; V.out_values = values;
  const int64_t m = (int64_t)n * top_k;
  if (m <= 0) return NRTGPU_OK;
  sort_fields_values_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(V);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// A searcher's leaf: the FieldDoc values [n][n_fields] of its hits, whose KEYWORD codes number the leaf's dictionary, to
// codes of the reader-wide union (sort_kw_map_kernel), before the leaves' records merge. maps: per field, NULL where
// nothing maps (see SortKwMapLaunch); nothing runs when every entry is NULL.
static int sort_kw_values_to_union(const uint32_t* const* maps, int n_fields, int64_t* values, int64_t n, cudaStream_t st) {
  SortKwMapLaunch M{};
  bool any = false;
  for (int j = 0; j < n_fields; ++j) { M.map[j] = maps[j]; any |= maps[j] != nullptr; }
  if (!any || n <= 0) return NRTGPU_OK;
  M.values = values; M.n = n; M.n_fields = n_fields;
  sort_kw_map_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// Nested top hits of terms or filter aggregation `parent` (pass 2) over the batches bs[0 .. n_b) that counted into one set of tables
// (a single image: one batch; a searcher: one per leaf). Each batch's engine runs again (batch_engine_launch: the probe
// kernel, or the window engine for tree and wide batches) with a collector that only
// appends the key of each doc of a returned bucket (slot map nest_slot) to per-(query, slot) segments sized by the bucket
// counts h_cnt [nq*size]: make_key(score, global doc), or for a sorted collector its Sort key over that leaf's order
// (agg_nested_collect); its totalHits / pruned / terminated go to scratch, and theta / slice lists / queue heads are its
// own, already merged. Queries are taken in groups whose keys fit kNestedHitBudget; each group runs every batch's launch
// into the same segments, then selects once. Sorted keys of distinct leaves do not compare, so over several leaves a sorted
// collector's segments are reset before each leaf's launch, the leaf selects its own top_hits into a packed sorted record
// (one list per (query, slot)), and the leaves' records are merged as TopFieldDocs.merge does before start_hit is applied.
// Scratch and results are bs[0]'s.
static int batch_nested_top_hits(nrtgpu_batch* const* bs, int n_b, cudaStream_t st, int parent, const std::vector<int32_t>& h_cnt,
                                 const nrtgpu_nested_result* nres) {
  nrtgpu_batch* b = bs[0];
  const int nq = b->nq;
  const nrtgpu_aggregation& a = b->cb.aggs[(size_t)parent];
  const int size = a.size;
  std::vector<size_t> th;   // the parent's top-hits collectors (indices into cb.nested)
  for (size_t j = 0; j < b->cb.nested.size(); ++j)
    if (b->cb.nested[j].parent == parent && b->cb.nested[j].kind == NRTGPU_AGG_TOP_HITS) th.push_back(j);
  const int n_th = (int)th.size();
  // the order of collector k on batch l (NULL: by score)
  auto order_of = [&](int k, int l) -> const nrtgpu_sort_order* {
    const nrtgpu_nested_sort& so = b->cb.nested_sorts[th[(size_t)k]];
    return so.orders ? so.orders[l] : nullptr;
  };
  const bool merge = n_b > 1;   // several leaves: sorted collectors select per leaf, then merge
  std::vector<size_t> out_base((size_t)n_th + 1, 0), val_base((size_t)n_th + 1, 0);
  std::vector<long long> rec_q((size_t)n_th, 0);   // merge: bytes of a sorted collector's records per query of a group
  for (int k = 0; k < n_th; ++k) {
    const nrtgpu_nested_aggregation& n = b->cb.nested[th[(size_t)k]];
    const size_t nw = (size_t)nq * size * (size_t)(n.top_hits - n.start_hit);
    const nrtgpu_sort_order* o = order_of(k, 0);
    out_base[(size_t)k + 1] = out_base[(size_t)k] + nw;
    val_base[(size_t)k + 1] = val_base[(size_t)k] + (o ? nw * (size_t)o->n_fields : 0);
    if (o && merge) rec_q[(size_t)k] = (long long)(n_b + 1) * size * ((long long)n.top_hits * (1 + 2 * o->n_fields) + 4) * 4;
  }
  int rc;
  if ((rc = b->nest_docs.alloc(out_base.back())) || (rc = b->nest_scores.alloc(out_base.back())) ||
      (rc = b->nest_svals.alloc(std::max<size_t>(val_base.back(), 1))) ||
      (rc = b->nest_hcounts.alloc((size_t)n_th * nq * size)) || (rc = b->p2_total.alloc((size_t)nq)) || (rc = b->p2_flags.alloc(2 * (size_t)nq)))
    return rc;
  std::vector<long long> per_q((size_t)nq, 0);
  for (int q = 0; q < nq; ++q)
    for (int s = 0; s < size; ++s) per_q[(size_t)q] += (long long)n_th * h_cnt[(size_t)q * size + s];
  long long rec_per_q = 0;
  for (long long x : rec_q) rec_per_q += x;
  for (int q_lo = 0; q_lo < nq;) {
    if (per_q[(size_t)q_lo] > kNestedHitBudget)
      NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nested top hits: the returned buckets of one query hold more than 2^26 hits");
    long long total = 0;
    int q_hi = q_lo;
    // (the sorted records of a group stay under 512 MB too, unless one query needs more by itself)
    while (q_hi < nq && total + per_q[(size_t)q_hi] <= kNestedHitBudget &&
           (q_hi == q_lo || (q_hi - q_lo + 1) * rec_per_q <= kNestedHitBudget * 8))
      total += per_q[(size_t)q_hi++];
    const int gq = q_hi - q_lo, gs = gq * size;
    std::vector<long long> off((size_t)n_th * (gs + 1));   // per collector: the segments of the group, laid out one after the other
    long long at = 0;
    for (int k = 0; k < n_th; ++k)
      for (int g = 0; g <= gs; ++g) {
        off[(size_t)k * (gs + 1) + g] = at;
        if (g < gs) at += h_cnt[(size_t)q_lo * size + g];
      }
    if ((rc = b->nest_off.upload_async(off.data(), off.size(), st)) || (rc = b->nest_fill.alloc((size_t)n_th * gs)) ||
        (rc = b->nest_keys.alloc((size_t)std::max(at, 1ll)))) return rc;
    NRT_CUDA_TRY(cudaMemsetAsync(b->nest_fill.p, 0, b->nest_fill.bytes(), st));
    // merge: per sorted collector, n_b leaf records then the merged one (int32 words; every record starts 8-byte aligned)
    std::vector<SortedRecordLayout> rl((size_t)n_th);
    std::vector<size_t> rec_at((size_t)n_th + 1, 0);
    int k_max = 1;
    for (int k = 0; k < n_th; ++k) {
      const nrtgpu_sort_order* o = order_of(k, 0);
      rec_at[(size_t)k + 1] = rec_at[(size_t)k];
      if (!o || !merge) continue;
      const int K = b->cb.nested[th[(size_t)k]].top_hits;
      rl[(size_t)k] = sorted_record_layout(gs, K, o->n_fields);
      rec_at[(size_t)k + 1] += (size_t)(n_b + 1) * (size_t)rl[(size_t)k].words;
      k_max = std::max(k_max, K);
    }
    if (rec_at.back() > 0) {
      if ((rc = b->nest_rec.alloc(rec_at.back() / 2)) || (rc = b->nest_rscores.alloc((size_t)gs * k_max))) return rc;
      NRT_CUDA_TRY(cudaMemsetAsync(b->nest_rec.p, 0, rec_at.back() * 4, st));
    }
    int32_t* rec = reinterpret_cast<int32_t*>(b->nest_rec.p);
    std::vector<AggLaunch> launches((size_t)n_b);   // uploaded asynchronously: kept until the group's synchronize
    for (int l = 0; l < n_b && at > 0; ++l) {
      nrtgpu_batch* x = bs[l];
      if (merge)   // this leaf's sorted keys start from empty segments
        for (int k = 0; k < n_th; ++k)
          if (order_of(k, l)) NRT_CUDA_TRY(cudaMemsetAsync(b->nest_fill.p + (size_t)k * gs, 0, (size_t)gs * sizeof(unsigned int), st));
      if (x->plan.n_work() > 0) {
        AggLaunch& A = launches[(size_t)l];
        std::memset(&A, 0, sizeof(A));
        A.n_aggs = 1;
        A.a[0].kind = NRTGPU_AGG_TERMS; A.a[0].column = a.kind == NRTGPU_AGG_FILTER || agg_keyword(a) ? x->ix->n_columns : a.column;
        A.a[0].value_type = a.value_type;
        A.a[0].n_buckets = x->agg_tab.n_buckets[parent];
        A.codes[0] = x->agg_codes[parent];   // the codes pass 1 counted through; counts stay NULL: the pass-1 tables are not touched
        A.offsets[0] = x->agg_tab.offsets[parent];
        A.nested_begin[1] = n_th;
        for (int k = 0; k < n_th; ++k) {
          AggNestedDev& d = A.nested[k];
          d.kind = NRTGPU_AGG_TOP_HITS; d.size = size; d.q_lo = q_lo; d.q_hi = q_hi; d.slot_of = b->nest_slot.p;
          d.hit_off = b->nest_off.p + (size_t)k * (gs + 1); d.hit_fill = b->nest_fill.p + (size_t)k * gs; d.hit_keys = b->nest_keys.p;
          d.doc_base = x->ix->doc_base; d.score_key = 1;
          if (const nrtgpu_sort_order* o = order_of(k, l)) { d.rank = o->rank.p; d.score_key = o->score_first; d.score_reverse = o->score_reverse; }
        }
        if ((rc = x->nest_launch.upload_async(&A, 1, st))) return rc;
        NRT_CUDA_TRY(cudaMemsetAsync(x->theta.p, 0, x->theta.bytes(), st));
        NRT_CUDA_TRY(cudaMemsetAsync(x->slice_cnt.p, 0, x->slice_cnt.bytes(), st));
        if (x->work_counter.p) NRT_CUDA_TRY(cudaMemsetAsync(x->work_counter.p, 0, x->work_counter.bytes(), st));   // (probe batches)
        NRT_CUDA_TRY(cudaMemsetAsync(b->p2_total.p, 0, b->p2_total.bytes(), st));
        NRT_CUDA_TRY(cudaMemsetAsync(b->p2_flags.p, 0, b->p2_flags.bytes(), st));
        if ((rc = batch_engine_launch(x, x->nest_launch.p, A.offsets[0] != nullptr, b->p2_total.p, b->p2_flags.p, false, st))) return rc;
      }
      for (int k = 0; k < n_th && merge; ++k) {   // this leaf's best top_hits of each list, by its order, into its record
        const nrtgpu_sort_order* o = order_of(k, l);
        if (!o) continue;
        const SortedRecordLayout& L = rl[(size_t)k];
        int32_t* r = rec + rec_at[(size_t)k] + (size_t)l * L.words;
        NestedHitsLaunch H;
        H.hit_keys = b->nest_keys.p; H.hit_off = b->nest_off.p + (size_t)k * (gs + 1); H.hit_fill = b->nest_fill.p + (size_t)k * gs;
        H.q_lo = 0; H.size = size; H.top_hits = b->cb.nested[th[(size_t)k]].top_hits; H.start_hit = 0; H.doc_base = x->ix->doc_base;
        H.out_docs = r; H.out_scores = b->nest_rscores.p; H.out_counts = r + L.counts;
        nested_top_hits_kernel<<<gs, 256, 0, st>>>(H);
        NRT_CUDA_TRY(cudaGetLastError());
        if ((rc = sorted_hit_values(o, x->ix->doc_base, r, r + L.counts, b->nest_rscores.p, gs, H.top_hits,
                                    reinterpret_cast<int64_t*>(r + L.values), st))) return rc;
        if (!x->nest_kw_map.empty() &&   // keyword values in the reader-wide dictionary, so the leaves' lists merge
            (rc = sort_kw_values_to_union(x->nest_kw_map[th[(size_t)k]].data(), o->n_fields, reinterpret_cast<int64_t*>(r + L.values),
                                          (int64_t)gs * H.top_hits, st))) return rc;
      }
    }
    for (int k = 0; k < n_th; ++k) {
      const nrtgpu_nested_aggregation& n = b->cb.nested[th[(size_t)k]];
      const nrtgpu_sort_order* o = order_of(k, 0);
      if (o && merge) {   // TopFieldDocs.merge of the leaves' lists, then positions [start_hit, top_hits)
        const SortedRecordLayout& L = rl[(size_t)k];
        int32_t* r = rec + rec_at[(size_t)k];
        if ((rc = nrtgpu_merge_sorted_packed(b->ix->ctx, o->spec, o->n_fields, n_b, gs, n.top_hits, r, r + (size_t)n_b * L.words, st)))
          return rc;
        SortedHitsOutLaunch S;
        S.record = r + (size_t)n_b * L.words; S.L = L; S.n = gs; S.top_k = n.top_hits; S.n_fields = o->n_fields;
        S.start_hit = n.start_hit; S.w = n.top_hits - n.start_hit; S.q_lo = q_lo; S.size = size;
        S.out_docs = b->nest_docs.p + out_base[(size_t)k]; S.out_scores = b->nest_scores.p + out_base[(size_t)k];
        S.out_counts = b->nest_hcounts.p + (size_t)k * nq * size; S.out_values = b->nest_svals.p + val_base[(size_t)k];
        const int m = gs * S.w;
        sorted_hits_out_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(S);
        NRT_CUDA_TRY(cudaGetLastError());
        continue;
      }
      NestedHitsLaunch H;
      H.hit_keys = b->nest_keys.p; H.hit_off = b->nest_off.p + (size_t)k * (gs + 1); H.hit_fill = b->nest_fill.p + (size_t)k * gs;
      H.q_lo = q_lo; H.size = size; H.top_hits = n.top_hits; H.start_hit = n.start_hit;
      H.doc_base = o ? b->ix->doc_base : 0;   // score keys hold global docs; Sort keys the image's ranks
      H.out_docs = b->nest_docs.p + out_base[(size_t)k]; H.out_scores = b->nest_scores.p + out_base[(size_t)k];
      H.out_counts = b->nest_hcounts.p + (size_t)k * nq * size;
      nested_top_hits_kernel<<<gs, 256, 0, st>>>(H);
      NRT_CUDA_TRY(cudaGetLastError());
    }
    NRT_CUDA_TRY(cudaStreamSynchronize(st));   // A and off are stack objects; the next group reuses the buffers
    q_lo = q_hi;
  }
  for (int k = 0; k < n_th; ++k) {
    const size_t j = th[(size_t)k];
    const nrtgpu_nested_result& r = nres[j];
    const size_t nw = out_base[(size_t)k + 1] - out_base[(size_t)k];
    const nrtgpu_sort_order* o = order_of(k, 0);
    if (o && !merge && (rc = sorted_hit_values(o, b->ix->doc_base, b->nest_docs.p + out_base[(size_t)k], b->nest_hcounts.p + (size_t)k * nq * size,
                                               b->nest_scores.p + out_base[(size_t)k], nq * size,
                                               b->cb.nested[j].top_hits - b->cb.nested[j].start_hit, b->nest_svals.p + val_base[(size_t)k], st)))
      return rc;
    if (r.hit_docs) NRT_CUDA_TRY(cudaMemcpyAsync(r.hit_docs, b->nest_docs.p + out_base[(size_t)k], nw * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (r.hit_scores) NRT_CUDA_TRY(cudaMemcpyAsync(r.hit_scores, b->nest_scores.p + out_base[(size_t)k], nw * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (r.hit_counts) NRT_CUDA_TRY(cudaMemcpyAsync(r.hit_counts, b->nest_hcounts.p + (size_t)k * nq * size, (size_t)nq * size * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (o && b->cb.nested_sorts[j].values)
      NRT_CUDA_TRY(cudaMemcpyAsync(b->cb.nested_sorts[j].values, b->nest_svals.p + val_base[(size_t)k],
                                   (val_base[(size_t)k + 1] - val_base[(size_t)k]) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    if (r.hit_total) for (size_t x = 0; x < (size_t)nq * size; ++x) r.hit_total[x] = h_cnt[x];   // TopDocs.totalHits: the bucket's count
  }
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  return NRTGPU_OK;
}

// aggregation results of the last run of the batches bs[0 .. n_b), which counted into one set of tables (agg_tab) ->
// caller buffers (nres: the results of cb.nested, in request order; NULL: none). The selection runs once on those tables.
static int batch_fetch_aggs(nrtgpu_batch* const* bs, int n_b, cudaStream_t st, const nrtgpu_aggregation_result* out,
                            const nrtgpu_nested_result* nres) {
  nrtgpu_batch* b = bs[0];
  const AggTables& t = b->agg_tab;
  const int nq = b->nq;
  for (size_t i = 0; i < b->cb.aggs.size(); ++i) {
    const nrtgpu_aggregation& a = b->cb.aggs[i];
    const nrtgpu_aggregation_result& r = out[i];
    if (a.kind == NRTGPU_AGG_TERMS || a.kind == NRTGPU_AGG_FILTER) {
      const bool filter = a.kind == NRTGPU_AGG_FILTER;   // one bucket per query (size 1): its count is the docCount
      int rc;
      const size_t n = (size_t)nq * a.size;
      if ((rc = b->agg_keys.alloc(n)) || (rc = b->agg_cnts.alloc(n)) || (rc = b->agg_n.alloc((size_t)nq)) || (rc = b->agg_tot.alloc((size_t)nq)) ||
          (rc = b->agg_other.alloc((size_t)nq))) return rc;
      int n_nested = 0, order_by = -1;
      bool top_hits = false;
      for (size_t j = 0; j < b->cb.nested.size(); ++j)
        if (b->cb.nested[j].parent == (int32_t)i) {
          ++n_nested;
          if (b->cb.nested[j].orders_parent) order_by = (int)j;
          top_hits |= b->cb.nested[j].kind == NRTGPU_AGG_TOP_HITS;
        }
      AggTermsLaunch T;
      T.counts = t.counts[i]; T.n_buckets = t.n_buckets[i]; T.nq = nq; T.size = a.size; T.order_desc = a.order_desc != 0;
      T.distinct = t.distinct[i];
      T.out_keys = b->agg_keys.p; T.out_counts = b->agg_cnts.p; T.out_n = b->agg_n.p; T.out_total_buckets = b->agg_tot.p; T.out_other = b->agg_other.p;
      T.out_bucket = nullptr;
      if (n_nested > 0) {
        if ((rc = b->agg_bucket.alloc(n))) return rc;
        T.out_bucket = b->agg_bucket.p;
      }
      if (filter) {
        NRT_CUDA_TRY(cudaMemcpyAsync(b->agg_cnts.p, t.counts[i], n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
        if (T.out_bucket) NRT_CUDA_TRY(cudaMemsetAsync(T.out_bucket, 0, n * sizeof(int32_t), st));
      } else if (order_by >= 0) {
        NRT_CUDA_TRY(cudaFuncSetAttribute(agg_terms_by_value_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAggByValueSmem));
        agg_terms_by_value_kernel<<<nq, 256, kAggByValueSmem, st>>>(T, t.nest_words[(size_t)order_by], b->cb.nested[(size_t)order_by].kind);
      } else {
        agg_terms_topk_kernel<<<nq, 256, 0, st>>>(T);
      }
      NRT_CUDA_TRY(cudaGetLastError());
      std::vector<int32_t> h_cnt;
      if (n_nested > 0) {   // per returned slot: nested values, the slot map of the top-hits run
        AggNestedOutLaunch O; std::memset(&O, 0, sizeof(O));
        O.bucket = b->agg_bucket.p; O.nq = nq; O.size = a.size; O.n_buckets = T.n_buckets;
        std::vector<size_t> vals;   // the min / max / sum collectors (indices into cb.nested)
        for (size_t j = 0; j < b->cb.nested.size(); ++j)
          if (b->cb.nested[j].parent == (int32_t)i && b->cb.nested[j].kind != NRTGPU_AGG_TOP_HITS) vals.push_back(j);
        if ((rc = b->nest_vals.alloc(std::max<size_t>(vals.size(), 1) * n))) return rc;
        O.n_vals = (int32_t)vals.size();
        for (size_t k = 0; k < vals.size(); ++k) {
          O.kind[k] = b->cb.nested[vals[k]].kind; O.words[k] = t.nest_words[vals[k]]; O.values[k] = b->nest_vals.p + k * n;
        }
        if (top_hits) {
          const size_t cells = (size_t)nq * (size_t)std::max(T.n_buckets, 1);
          if ((rc = b->nest_slot.alloc(cells))) return rc;
          NRT_CUDA_TRY(cudaMemsetAsync(b->nest_slot.p, 0xff, cells * sizeof(int32_t), st));
          O.slot_of = b->nest_slot.p;
        }
        agg_nested_out_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(O);
        NRT_CUDA_TRY(cudaGetLastError());
        for (size_t k = 0; k < vals.size(); ++k)
          if (nres && nres[vals[k]].values)
            NRT_CUDA_TRY(cudaMemcpyAsync(nres[vals[k]].values, b->nest_vals.p + k * n, n * sizeof(double), cudaMemcpyDeviceToHost, st));
        h_cnt.resize(n);
        NRT_CUDA_TRY(cudaMemcpyAsync(h_cnt.data(), b->agg_cnts.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      }
      if (r.bucket_counts) NRT_CUDA_TRY(cudaMemcpyAsync(r.bucket_counts, b->agg_cnts.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      if (!filter) {   // (a filter's docCount is its only result)
        if (r.bucket_keys) NRT_CUDA_TRY(cudaMemcpyAsync(r.bucket_keys, b->agg_keys.p, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        if (r.n_buckets) NRT_CUDA_TRY(cudaMemcpyAsync(r.n_buckets, b->agg_n.p, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (r.total_buckets) NRT_CUDA_TRY(cudaMemcpyAsync(r.total_buckets, b->agg_tot.p, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (r.other_counts) NRT_CUDA_TRY(cudaMemcpyAsync(r.other_counts, b->agg_other.p, (size_t)nq * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
      }
      NRT_CUDA_TRY(cudaStreamSynchronize(st));   // the scratch is reused by the next terms aggregation
      if (top_hits && (rc = batch_nested_top_hits(bs, n_b, st, (int)i, h_cnt, nres))) return rc;
    } else if (r.values) {
      std::vector<unsigned long long> h((size_t)nq);
      NRT_CUDA_TRY(cudaMemcpyAsync(h.data(), t.dvals[i], (size_t)nq * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      NRT_CUDA_TRY(cudaStreamSynchronize(st));
      for (int q = 0; q < nq; ++q) r.values[q] = agg_word_value(a.kind, h[(size_t)q]);
    }
  }
  return NRTGPU_OK;
}

// deadline / terminateAfter of the batch (SearchCutoffWrapper / TerminateAfterWrapper semantics, see include/nrtgpu.h)
static int batch_set_limits(nrtgpu_batch* b, const nrtgpu_search_limits* lim, cudaStream_t st) {
  b->limits_active = false; b->disallow_partial = false; b->timeout_sec = 0.0; b->terminate_after_max_recall = 0;
  b->deadline_ns = 0; b->ta_scalar = 0;
  if (!lim) return NRTGPU_OK;
  if (lim->timeout_sec < 0.0 || lim->terminate_after < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "timeout_sec / terminate_after must be >= 0");
  int rc;
  if (lim->timeout_sec > 0.0) {
    b->limits_active = true; b->timeout_sec = lim->timeout_sec; b->disallow_partial = lim->disallow_partial_results != 0;
    const double left = lim->timeout_sec - lim->elapsed_sec;   // the timer started when the request's first collector was created
    b->deadline_ns = left <= 0.0 ? -1 : std::max<long long>(1, (long long)(left * 1e9));
    if ((rc = b->timed_out.alloc((size_t)b->nq))) return rc;
    if ((rc = b->clock0.alloc(1))) return rc;
  }
  if (lim->terminate_after > 0) {
    b->ta_scalar = lim->terminate_after;
    b->terminate_after_max_recall = lim->terminate_after_max_recall_count > lim->terminate_after ? lim->terminate_after_max_recall_count : lim->terminate_after;
  }
  (void)st;
  return NRTGPU_OK;
}

int nrtgpu_batch_set_limits(nrtgpu_batch* b, const nrtgpu_search_limits* limits) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  return batch_set_limits(b, limits, (cudaStream_t)0);
}

int nrtgpu_batch_device_results(nrtgpu_batch* b, int32_t** d_docs, float** d_scores, int32_t** d_counts) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  if (d_docs) *d_docs = b->o_docs();
  if (d_scores) *d_scores = b->o_scores();
  if (d_counts) *d_counts = b->o_counts();
  return NRTGPU_OK;
}

int nrtgpu_batch_bind_output(nrtgpu_batch* b, int32_t* d_docs, float* d_scores, int32_t* d_counts) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  b->bound_docs = d_docs; b->bound_scores = d_scores; b->bound_counts = d_counts;
  b->bound_total = nullptr; b->bound_flags = nullptr; b->bound_values = nullptr;
  return NRTGPU_OK;
}

// Packed per-shard result record (one all-gather carries everything TopDocs.merge needs), int32 words:
//   docs [nq*top_k] | scores [nq*top_k] (float bits) | counts [nq] | flags [nq] | (pad to 8 bytes) | totalHits [nq] int64
int64_t nrtgpu_packed_words(int32_t nq, int32_t top_k) {
  int64_t w = (int64_t)nq * top_k * 2 + 2ll * nq;
  w = (w + 1) & ~1ll;
  return w + 2ll * nq;
}

int nrtgpu_batch_bind_packed(nrtgpu_batch* b, int32_t* d_record) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  if (!d_record) { b->unbind(); return NRTGPU_OK; }
  if (((uintptr_t)d_record & 7u) != 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_bind_packed: record must be 8-byte aligned");
  const int64_t n = (int64_t)b->nq * b->top_k;
  b->bound_values = nullptr;
  b->bound_docs = d_record; b->bound_scores = (float*)(d_record + n); b->bound_counts = d_record + 2 * n;
  b->bound_flags = d_record + 2 * n + b->nq;
  int64_t w = 2 * n + 2ll * b->nq; w = (w + 1) & ~1ll;
  b->bound_total = (long long*)(d_record + w);
  return NRTGPU_OK;
}

int nrtgpu_merge_topk_packed(nrtgpu_ctx* ctx, int32_t n_lists, int32_t nq, int32_t top_k, const int32_t* d_records,
                             int32_t* d_out_record, void* stream) {
  if (!ctx || !d_records || !d_out_record || n_lists <= 0 || nq <= 0 || top_k <= 0 || top_k > kMaxTopK)
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_topk_packed: bad argument");
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  const int64_t n = (int64_t)nq * top_k, words = nrtgpu_packed_words(nq, top_k);
  int64_t w = 2 * n + 2ll * nq; w = (w + 1) & ~1ll;
  MergePairsLaunch M;
  M.docs = d_records; M.scores = (const float*)(d_records + n); M.counts = d_records + 2 * n;
  M.stride_hits = words; M.stride_counts = words;
  M.n_lists = n_lists; M.top_k = top_k; M.nq = nq;
  M.out_docs = d_out_record; M.out_scores = (float*)(d_out_record + n); M.out_counts = d_out_record + 2 * n;
  M.flags = d_records + 2 * n + nq; M.totals = (const long long*)(d_records + w); M.stride_flags = words; M.stride_totals = words / 2;
  M.out_flags = d_out_record + 2 * n + nq; M.out_total = (long long*)(d_out_record + w);
  merge_pairs_kernel<<<nq, kMergeThreads, 0, (cudaStream_t)stream>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

int nrtgpu_batch_reset_timing(nrtgpu_batch* b) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  b->runs_recorded = 0;
  return NRTGPU_OK;
}

int nrtgpu_batch_stats(const nrtgpu_batch* b, int64_t* alg_postings, int32_t* launches_per_run, int64_t* work_items) {
  if (!b) NRT_FAIL(NRTGPU_ERR_INVALID, "NULL batch");
  if (alg_postings) *alg_postings = b->cb.alg_postings;
  if (launches_per_run) {
    int n = 1;   // slice merge
    if (b->cb.wide) n += b->plan.n_work() > 0 ? 1 : 0;
    else n += (b->plan.n_probe_simple > 0 ? 1 : 0) + (b->plan.n_probe_generic > 0 ? 1 : 0);
    *launches_per_run = n;
  }
  if (work_items) *work_items = b->plan.n_work();
  return NRTGPU_OK;
}

int nrtgpu_batch_stage_ms(nrtgpu_batch* b, int32_t stage, float* ms) {
  if (!b || !ms || stage < 0 || stage > 1 || !b->ran || b->runs_recorded < 1) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_batch_stage_ms: bad argument");
  int n = std::min(b->runs_recorded, (int)nrtgpu_batch::kEvRing);
  double sum = 0.0;
  for (int i = 0; i < n; ++i) {
    float t = 0.f;
    NRT_CUDA_TRY(cudaEventElapsedTime(&t, b->ev[i][stage], b->ev[i][stage + 1]));
    sum += t;
  }
  *ms = (float)(sum / n);
  return NRTGPU_OK;
}

int nrtgpu_batch_free(nrtgpu_batch* b) {
  if (b) { cudaSetDevice(b->ix->ctx->device); delete b; }
  return NRTGPU_OK;
}

// redirects the results of subsequent runs of a sort-order batch into a sorted record (sorted_record_layout); the scores the
// score-first key needs stay in the batch's own buffer
static int batch_bind_sorted(nrtgpu_batch* b, int32_t* d_record, int32_t n_fields) {
  if (((uintptr_t)d_record & 7u) != 0) NRT_FAIL(NRTGPU_ERR_INVALID, "sorted record must be 8-byte aligned");
  if (!b->order || n_fields <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "a sorted record needs a sort order");
  const SortedRecordLayout L = sorted_record_layout(b->nq, b->top_k, n_fields);
  b->unbind();
  b->bound_docs = d_record; b->bound_counts = d_record + L.counts; b->bound_flags = d_record + L.flags;
  b->bound_total = (long long*)(d_record + L.totals); b->bound_values = (int64_t*)(d_record + L.values);
  return NRTGPU_OK;
}

// a pooled batch workspace of the index (device buffers survive between calls: no cudaMalloc on the request path), checked
// out for one call; returned with its bound outputs cleared
struct WorkspaceLease {
  nrtgpu_index* ix;
  nrtgpu_batch* b = nullptr;
  explicit WorkspaceLease(nrtgpu_index* ix_) : ix(ix_) {
    { std::lock_guard<std::mutex> g(ix->ws_mu); if (!ix->ws_free.empty()) { b = ix->ws_free.back(); ix->ws_free.pop_back(); } }
    if (!b) b = new nrtgpu_batch;
  }
  ~WorkspaceLease() { b->unbind(); std::lock_guard<std::mutex> g(ix->ws_mu); ix->ws_free.push_back(b); }
  WorkspaceLease(const WorkspaceLease&) = delete;
  WorkspaceLease& operator=(const WorkspaceLease&) = delete;
};

// where a one-shot search leaves its results: a packed DEVICE record (the multi-GPU path: the caller all-gathers it on
// the stream), a packed sorted DEVICE record (d_sorted_record, searches with a sort order), or else the HOST buffers (any
// may be NULL). record_limits: a record also carries what batch_fetch_impl derives from the limits on the host (hit_timeout
// as flags bit 2 and relation GTE, the terminateAfterMaxRecallCount cap, and NRTGPU_ERR_TIMEOUT with disallow_partial_results).
struct SearchOut {
  int32_t* d_record = nullptr;
  int32_t* d_sorted_record = nullptr;
  bool record_limits = false;
  int32_t* docs = nullptr; float* scores = nullptr; int32_t* counts = nullptr; int64_t* total_hits = nullptr;
  uint8_t* relation = nullptr; uint8_t* hit_timeout = nullptr; uint8_t* terminated_early = nullptr;
  int64_t* sort_values = nullptr;
  const nrtgpu_aggregation_result* aggs = nullptr;
  const nrtgpu_nested_result* nested = nullptr;
};

// one-shot search: compile + upload the batch into a pooled workspace, run, deliver the results
static int search_bool_impl(nrtgpu_index* ix, const BatchRequest& r, const nrtgpu_search_limits* limits, void* stream, const SearchOut& out) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_bool: NULL index");
  WorkspaceLease ws(ix);
  nrtgpu_batch* b = ws.b;
  int rc = batch_build(b, ix, r, (cudaStream_t)stream);
  if (!rc) rc = batch_set_limits(b, limits, (cudaStream_t)stream);
  if (!rc && out.d_record) rc = nrtgpu_batch_bind_packed(b, out.d_record);
  if (!rc && out.d_sorted_record) rc = batch_bind_sorted(b, out.d_sorted_record, r.sort_order ? r.sort_order->n_fields : 0);
  if (!rc) rc = nrtgpu_batch_run(b, stream);
  if (rc) return rc;
  if (out.d_record || out.d_sorted_record) {
    cudaStream_t st = (cudaStream_t)stream;
    if (out.record_limits && (b->limits_active || b->terminate_after_max_recall > 0)) {
      record_limits_kernel<<<(unsigned)((r.nq + 127) / 128), 128, 0, st>>>(r.nq, b->limits_active ? b->timed_out.p : nullptr,
                                                                          b->terminate_after_max_recall, b->bound_flags, b->bound_total);
      NRT_CUDA_TRY(cudaGetLastError());
    }
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return NRTGPU_ERR_CUDA; }
    if (out.record_limits && b->limits_active && b->disallow_partial) {
      std::vector<int32_t>& to = b->h_flags;
      to.resize((size_t)r.nq);
      NRT_CUDA_TRY(cudaMemcpy(to.data(), b->timed_out.p, (size_t)r.nq * sizeof(int32_t), cudaMemcpyDeviceToHost));
      for (int q = 0; q < r.nq; ++q)
        if (to[(size_t)q]) NRT_FAIL(NRTGPU_ERR_TIMEOUT, "Search collection exceeded timeout of " + std::to_string(b->timeout_sec) + "s");
    }
    return NRTGPU_OK;
  }
  if (out.sort_values && b->sort_kind != NRTGPU_SORT_RELEVANCE) {
    const size_t nv = (size_t)r.nq * r.top_k * (r.sort_order ? r.sort_order->n_fields : 1);
    cudaError_t e = cudaMemcpyAsync(out.sort_values, b->out_sort_values.p, nv * sizeof(int64_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return NRTGPU_ERR_CUDA; }
  }
  rc = batch_fetch_impl(b, stream, out.docs, out.scores, out.counts, out.total_hits, out.relation, out.hit_timeout, out.terminated_early);
  if (!rc && !b->cb.aggs.empty() && out.aggs) rc = batch_fetch_aggs(&b, 1, (cudaStream_t)stream, out.aggs, out.nested);
  return rc;
}

int nrtgpu_search_bool(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                       const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                       int32_t total_hits_threshold, int32_t flags, void* stream, int32_t* out_docs,
                       float* out_scores, int32_t* out_counts, int64_t* out_total_hits,
                       uint8_t* out_relation) {
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  return search_bool_impl(ix, BatchRequest{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags}, nullptr, stream, o);
}

int nrtgpu_search_bool_ex(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                          const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                          const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores,
                          int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                          uint8_t* out_terminated_early) {
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  o.hit_timeout = out_hit_timeout; o.terminated_early = out_terminated_early;
  return search_bool_impl(ix, BatchRequest{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags}, limits, stream, o);
}

// a request of the tree entry points; without nodes it is the flat request of nrtgpu_search_bool_ex
static BatchRequest tree_request(const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                                 const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags) {
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags};
  if (n_nodes > 0) { r.nodes = nodes; r.n_nodes = n_nodes; }
  r.joins = true;
  return r;
}

int nrtgpu_search_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                       const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                       const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                       int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  o.hit_timeout = out_hit_timeout; o.terminated_early = out_terminated_early;
  return search_bool_impl(ix, tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, total_hits_threshold, flags), limits, stream, o);
}

// the phrase table of the phrase entry points; without phrases the request stays that of nrtgpu_search_tree
static int phrase_request(BatchRequest* r, const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms,
                          int32_t n_phrase_terms) {
  if (n_phrases < 0 || n_phrase_terms < 0 || (n_phrases > 0 && !phrases) || (n_phrase_terms > 0 && !phrase_terms))
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree_phrases: bad phrases");
  if (n_phrases > 0) { r->phrases = phrases; r->n_phrases = n_phrases; r->phrase_terms = phrase_terms; r->n_phrase_terms = n_phrase_terms; }
  return NRTGPU_OK;
}

int nrtgpu_search_tree_phrases(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                               int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                               const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                               int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                               const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores,
                               int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                               uint8_t* out_terminated_early) {
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  BatchRequest r = tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, total_hits_threshold, flags);
  int rc = phrase_request(&r, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc) return rc;
  r.unions = true;
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  o.hit_timeout = out_hit_timeout; o.terminated_early = out_terminated_early;
  return search_bool_impl(ix, r, limits, stream, o);
}

int nrtgpu_search_sorted(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                         const nrtgpu_sort* sort, const nrtgpu_search_limits* limits, void* stream,
                         int32_t* out_docs, int64_t* out_sort_values, int32_t* out_counts,
                         int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                         uint8_t* out_terminated_early) {
  if (!sort) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_sorted: NULL sort");
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, flags};
  r.sort = sort;
  SearchOut o; o.docs = out_docs; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  o.hit_timeout = out_hit_timeout; o.terminated_early = out_terminated_early; o.sort_values = out_sort_values;
  return search_bool_impl(ix, r, limits, stream, o);
}

int nrtgpu_sort_order_create(nrtgpu_index* ix, const nrtgpu_sort_field* fields, int32_t n_fields, void* stream, nrtgpu_sort_order** out) {
  if (!ix || !fields || !out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_sort_order_create: NULL argument");
  if (n_fields < 1) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_sort_order_create: a Sort needs at least one field");
  if (n_fields > kMaxSortFields) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nrtgpu_sort_order_create: more than 8 sort fields is not on the GPU path");
  std::unique_ptr<nrtgpu_sort_order> o(new nrtgpu_sort_order);
  o->ix = ix; o->n_fields = n_fields;
  for (int i = 0; i < n_fields; ++i) {
    const nrtgpu_sort_field& s = fields[i];
    SortFieldDev& f = o->f[i];
    o->spec[i] = s;
    f.kind = s.kind; f.reverse = s.reverse != 0; f.selector = s.selector; f.missing = s.missing_value;
    if (s.kind == NRTGPU_SORT_COLUMN) {
      if (s.column < 0 || s.column >= ix->n_columns) NRT_FAIL(NRTGPU_ERR_INVALID, "sort column out of range (field does not support sorting: no doc values)");
      if (s.selector != NRTGPU_SELECT_MIN && s.selector != NRTGPU_SELECT_MAX) NRT_FAIL(NRTGPU_ERR_INVALID, "bad sort selector");
      const size_t c = (size_t)s.column;
      if (ix->col_multi[c]) { f.mv_off = ix->colmv_off[c]->p; f.c64 = ix->col64[c]->p; }
      else {
        f.c64 = ix->col64[c]->p; f.c32 = ix->col32[c]->p; f.has = ix->col_has[c]->p;
        f.codes = ix->col_code[c]->p; f.distinct = ix->col_distinct[c]->p; f.n_distinct = ix->col_n_distinct[c];
      }
    } else if (s.kind == NRTGPU_SORT_KEYWORD) {
      if (s.column < 0 || (size_t)s.column >= ix->kw.size()) NRT_FAIL(NRTGPU_ERR_INVALID, "keyword sort column out of range");
      if (s.selector < NRTGPU_SELECT_MIN || s.selector > NRTGPU_SELECT_MIDDLE_MAX) NRT_FAIL(NRTGPU_ERR_INVALID, "bad sort selector");
      if (s.missing_value != 0 && s.missing_value != 1)
        NRT_FAIL(NRTGPU_ERR_INVALID, "keyword sort missing_value must be 0 (STRING_FIRST) or 1 (STRING_LAST)");
      const KeywordColumn& c = *ix->kw[(size_t)s.column];
      f.codes = c.codes.p; f.mv_off = c.multi ? c.doc_off.p : nullptr; f.n_distinct = c.n_terms;
    } else if (s.kind == NRTGPU_SORT_SCORE) {
      if (i > 0) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "a SCORE sort field is on the GPU path only in first position");
      o->score_first = true; o->score_reverse = s.reverse != 0;
    } else if (s.kind != NRTGPU_SORT_DOCID) NRT_FAIL(NRTGPU_ERR_INVALID, "bad sort field kind");
  }
  const int r0 = o->score_first ? 1 : 0;
  int r1 = n_fields;   // the fields after the first DOCID cannot decide anything
  for (int i = r0; i < n_fields; ++i) if (fields[i].kind == NRTGPU_SORT_DOCID) { r1 = i + 1; break; }
  o->n_rank = r1 - r0;
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  const int32_t n = ix->n_docs;
  int rc;
  if ((rc = o->perm.alloc((size_t)std::max(n, 1))) || (rc = o->rank.alloc((size_t)std::max(n, 1)))) return rc;
  o->perm.n = (size_t)n; o->rank.n = (size_t)n;
  {
    DevBuf<uint32_t> k32; DevBuf<uint64_t> k64;
    if ((rc = k32.alloc((size_t)std::max(n, 1))) || (rc = k64.alloc((size_t)std::max(n, 1)))) return rc;
    if ((rc = sort_order_build(o->f + r0, o->n_rank, n, ix->doc_base, (cudaStream_t)stream, o->perm.p, o->rank.p,
                               k32.p, k64.p))) return rc;
    NRT_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));   // the scratch is freed on return
  }
  *out = o.release();
  return NRTGPU_OK;
}

int64_t nrtgpu_sort_order_device_bytes(const nrtgpu_sort_order* o) { return o ? (int64_t)(o->perm.bytes() + o->rank.bytes()) : 0; }

int nrtgpu_sort_order_close(nrtgpu_sort_order* o) {
  if (!o) return NRTGPU_OK;
  cudaSetDevice(o->ix->ctx->device);
  delete o;
  return NRTGPU_OK;
}

int nrtgpu_search_sorted_fields(nrtgpu_index* ix, const nrtgpu_sort_order* order, const nrtgpu_clause* clauses, int32_t n_clauses,
                                const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags, const int64_t* after_values,
                                const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, int64_t* out_sort_values,
                                int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                                uint8_t* out_terminated_early) {
  if (!ix || !order) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_sorted_fields: NULL argument");
  if (order->ix != ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_sorted_fields: the sort order was made on another index");
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, flags};
  r.sort_order = order; r.order_after = after_values;
  SearchOut o; o.docs = out_docs; o.counts = out_counts; o.total_hits = out_total_hits; o.relation = out_relation;
  o.hit_timeout = out_hit_timeout; o.terminated_early = out_terminated_early; o.sort_values = out_sort_values;
  return search_bool_impl(ix, r, limits, stream, o);
}

int64_t nrtgpu_sorted_packed_words(int32_t nq, int32_t top_k, int32_t n_fields) {
  if (nq <= 0 || top_k <= 0 || n_fields < 1 || n_fields > kMaxSortFields) return 0;
  return sorted_record_layout(nq, top_k, n_fields).words;
}

int nrtgpu_search_sorted_fields_packed(nrtgpu_index* ix, const nrtgpu_sort_order* order, const nrtgpu_clause* clauses,
                                       int32_t n_clauses, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                       const int64_t* after_values, const nrtgpu_search_limits* limits, void* stream,
                                       int32_t* d_record) {
  if (!ix || !order || !d_record) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_sorted_fields_packed: NULL argument");
  if (order->ix != ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_sorted_fields_packed: the sort order was made on another index");
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, flags};
  r.sort_order = order; r.order_after = after_values;
  SearchOut o; o.d_sorted_record = d_record; o.record_limits = true;
  return search_bool_impl(ix, r, limits, stream, o);
}

int nrtgpu_merge_sorted_packed(nrtgpu_ctx* ctx, const nrtgpu_sort_field* fields, int32_t n_fields, int32_t n_lists, int32_t nq,
                               int32_t top_k, const int32_t* d_records, int32_t* d_out_record, void* stream) {
  if (!ctx || !fields || !d_records || !d_out_record) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_sorted_packed: NULL argument");
  if (n_lists < 1 || n_fields < 1 || n_fields > kMaxSortFields || nq <= 0 || top_k <= 0 || top_k > kMaxTopK)
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_sorted_packed: bad argument");
  if ((((uintptr_t)d_records | (uintptr_t)d_out_record) & 7u) != 0)
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_sorted_packed: records must be 8-byte aligned");
  SortMergeLaunch S{};
  S.records = d_records; S.out = d_out_record; S.L = sorted_record_layout(nq, top_k, n_fields);
  S.n_lists = n_lists; S.nq = nq; S.top_k = top_k; S.n_fields = n_fields; S.n_cmp = n_fields;
  for (int i = n_fields - 1; i >= 0; --i) {   // the fields after the first DOCID cannot decide anything
    const int32_t k = fields[i].kind;
    if (k != NRTGPU_SORT_COLUMN && k != NRTGPU_SORT_DOCID && k != NRTGPU_SORT_SCORE && k != NRTGPU_SORT_KEYWORD)
      NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_sorted_packed: bad sort field kind");
    if (k == NRTGPU_SORT_DOCID) S.n_cmp = i + 1;
    S.kind[i] = k; S.reverse[i] = fields[i].reverse != 0;
    if (k == NRTGPU_SORT_KEYWORD && fields[i].missing_value != 0) S.missing_last |= 1 << i;
  }
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  sort_merge_kernel<<<(unsigned)nq, kSortMergeThreads, 0, (cudaStream_t)stream>>>(S);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

int nrtgpu_search_bool_aggs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                            const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                            void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                            int64_t* out_total_hits) {
  return nrtgpu_search_bool_aggs_filtered(ix, clauses, n_clauses, queries, nq, top_k, flags, aggs, n_aggs, results, nullptr, 0, nullptr,
                                          nullptr, nullptr, 0, nullptr, 0, stream, out_docs, out_scores, out_counts, out_total_hits);
}

int nrtgpu_search_bool_aggs_nested(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                   const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                   const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                   const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                   const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs,
                                   float* out_scores, int32_t* out_counts, int64_t* out_total_hits) {
  return nrtgpu_search_bool_aggs_filtered(ix, clauses, n_clauses, queries, nq, top_k, flags, aggs, n_aggs, results, nested, n_nested,
                                          nested_results, nullptr, nullptr, 0, nullptr, 0, stream, out_docs, out_scores, out_counts,
                                          out_total_hits);
}

// the request of the additional-collector entry points (single image and searcher): exhaustive, with the collectors
static int aggs_request(BatchRequest* r, const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                        const nrtgpu_nested_aggregation* nested, int32_t n_nested, const nrtgpu_nested_result* nested_results,
                        const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                        int32_t n_filter_clauses, const nrtgpu_query* filter_queries, int32_t n_filter_queries) {
  if (n_aggs <= 0 || !aggs || !results) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_bool_aggs: no aggregations");
  if (n_nested < 0 || (n_nested > 0 && (!nested || !nested_results))) NRT_FAIL(NRTGPU_ERR_INVALID, "nested aggregations: NULL argument");
  if (n_filter_clauses < 0 || n_filter_queries < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "filter aggregation: negative filter query count");
  r->total_hits_threshold = INT32_MAX;
  r->aggs = aggs; r->n_aggs = n_aggs;
  if (n_nested > 0) { r->nested = nested; r->n_nested = n_nested; r->nested_sorts = nested_sorts; }
  r->agg_filters = agg_filters;
  r->filter_clauses = filter_clauses; r->n_filter_clauses = n_filter_clauses;
  r->filter_queries = filter_queries; r->n_filter_queries = n_filter_queries;
  return NRTGPU_OK;
}

static bool same_sort(const nrtgpu_sort_order* a, const nrtgpu_sort_order* b);

// the orders of the sorted top hits of a request (nested_sorts) on the images leaves[0 .. n_leaves): one per leaf, made on
// it, all of one Sort. An order on another kind of record is the compiler's refusal.
static int check_nested_sorts(const char* fn, const BatchRequest& r, nrtgpu_index* const* leaves, int n_leaves) {
  if (!r.nested_sorts) return NRTGPU_OK;
  const std::string f(fn);
  for (int j = 0; j < r.n_nested; ++j) {
    const nrtgpu_sort_order* const* orders = r.nested_sorts[j].orders;
    if (!orders || r.nested[j].kind != NRTGPU_AGG_TOP_HITS) continue;
    for (int l = 0; l < n_leaves; ++l) {
      if (!orders[l]) NRT_FAIL(NRTGPU_ERR_INVALID, f + ": NULL sort order");
      if (orders[l]->ix != leaves[l])
        NRT_FAIL(NRTGPU_ERR_INVALID, f + (n_leaves == 1 ? ": the sort order was made on another index"
                                                         : ": the sort order of leaf " + std::to_string(l) + " was made on another index"));
      if (!same_sort(orders[l], orders[0])) NRT_FAIL(NRTGPU_ERR_INVALID, f + ": the leaves' sort orders are of different Sorts");
    }
  }
  return NRTGPU_OK;
}

int nrtgpu_search_bool_aggs_filtered(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                     const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                     const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                     const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                     const nrtgpu_nested_result* nested_results, const nrtgpu_agg_filter* agg_filters,
                                     const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                                     const nrtgpu_query* filter_queries, int32_t n_filter_queries, void* stream,
                                     int32_t* out_docs, float* out_scores, int32_t* out_counts, int64_t* out_total_hits) {
  return nrtgpu_search_bool_aggs_sorted_hits(ix, clauses, n_clauses, queries, nq, top_k, flags, aggs, n_aggs, results, nested, n_nested,
                                             nested_results, nullptr, agg_filters, filter_clauses, n_filter_clauses, filter_queries,
                                             n_filter_queries, stream, out_docs, out_scores, out_counts, out_total_hits);
}

int nrtgpu_search_bool_aggs_sorted_hits(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                        const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                        const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                        const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                        const nrtgpu_nested_result* nested_results, const nrtgpu_nested_sort* nested_sorts,
                                        const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                        int32_t n_filter_clauses, const nrtgpu_query* filter_queries, int32_t n_filter_queries,
                                        void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                                        int64_t* out_total_hits) {
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, flags};
  int rc = aggs_request(&r, aggs, n_aggs, results, nested, n_nested, nested_results, nested_sorts, agg_filters, filter_clauses,
                        n_filter_clauses, filter_queries, n_filter_queries);
  if (rc || (rc = check_nested_sorts("nrtgpu_search_bool_aggs_sorted_hits", r, &ix, 1))) return rc;
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.aggs = results;
  o.nested = n_nested > 0 ? nested_results : nullptr;
  return search_bool_impl(ix, r, nullptr, stream, o);
}

// the request of the tree entry points with collectors: a tree (or flat) batch with the phrase table and the collectors of
// nrtgpu_search_bool_aggs_sorted_hits, collected by whichever engine runs the batch
static int tree_aggs_request(BatchRequest* r, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                             const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms,
                             int32_t n_phrase_terms, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                             const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                             const nrtgpu_nested_aggregation* nested, int32_t n_nested, const nrtgpu_nested_result* nested_results,
                             const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                             const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                             int32_t n_filter_queries) {
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  *r = tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, INT32_MAX, flags);
  int rc = phrase_request(r, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc || (rc = aggs_request(r, aggs, n_aggs, results, nested, n_nested, nested_results, nested_sorts, agg_filters, filter_clauses,
                               n_filter_clauses, filter_queries, n_filter_queries))) return rc;
  r->window_collectors = true;
  r->unions = true;
  return NRTGPU_OK;
}

int nrtgpu_search_tree_aggs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                            const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms,
                            int32_t n_phrase_terms, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                            const nrtgpu_nested_aggregation* nested, int32_t n_nested, const nrtgpu_nested_result* nested_results,
                            const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                            const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                            int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                            int64_t* out_total_hits) {
  BatchRequest r;
  int rc = tree_aggs_request(&r, clauses, n_clauses, nodes, n_nodes, phrases, n_phrases, phrase_terms, n_phrase_terms, queries, nq, top_k,
                             flags, aggs, n_aggs, results, nested, n_nested, nested_results, nested_sorts, agg_filters, filter_clauses,
                             n_filter_clauses, filter_queries, n_filter_queries);
  if (rc || (rc = check_nested_sorts("nrtgpu_search_tree_aggs", r, &ix, 1))) return rc;
  SearchOut o; o.docs = out_docs; o.scores = out_scores; o.counts = out_counts; o.total_hits = out_total_hits; o.aggs = results;
  o.nested = n_nested > 0 ? nested_results : nullptr;
  return search_bool_impl(ix, r, nullptr, stream, o);
}

// the request of the compile-only entry points: exhaustive, one hit per query (they never run the batch)
static BatchRequest compile_only_request(const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_query* queries, int32_t nq) {
  return BatchRequest{clauses, n_clauses, queries, nq, 1, INT32_MAX, 0};
}

// the second pass of a compiled request on the hit lists in b->sd_docs (b->sd_counts when counts is set): the flat
// score_docs_kernel, or score_docs_tree_kernel for a tree batch
static int launch_score_docs(nrtgpu_batch* b, nrtgpu_index* ix, int32_t nq, int32_t n_hits, bool counts, cudaStream_t st) {
  const size_t n = (size_t)nq * n_hits;
  int rc;
  if ((rc = b->sd_match.alloc(n)) || (rc = b->sd_scores.alloc(n))) return rc;
  ScoreDocsLaunch S; S.ix = ix->view(); S.clauses = b->clauses.p; S.queries = b->queries.p; S.nq = nq; S.n_hits = n_hits;
  S.docs = b->sd_docs.p; S.counts = counts ? b->sd_counts.p : nullptr; S.out_matches = b->sd_match.p; S.out_scores = b->sd_scores.p;
  if (!b->cb.tree) {
    score_docs_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(S);
  } else {
    ScoreDocsTreeLaunch T;
    static_cast<ScoreDocsLaunch&>(T) = S;
    T.nodes = b->nodes.p; T.node_begin = b->node_begin.p; T.phrases = b->phrases.p; T.phrase_begin = b->phrase_begin.p;
    T.n_chunks = (n_hits + kScoreTreeThreads - 1) / kScoreTreeThreads;
    if ((int64_t)T.n_chunks * nq > INT32_MAX) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "second pass: too many hits in one batch");
    score_docs_tree_kernel<<<(unsigned)(T.n_chunks * nq), kScoreTreeThreads, 0, st>>>(T);
  }
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// nrtgpu_score_docs / nrtgpu_score_docs_tree (fn names the entry point in messages)
static int score_docs_impl(const char* fn, nrtgpu_index* ix, const BatchRequest& r, int32_t n_hits, const int32_t* docs,
                           const int32_t* counts, void* stream, uint8_t* out_matches, float* out_scores) {
  if (!ix || !docs || !out_matches || !out_scores || n_hits <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  WorkspaceLease ws(ix);
  nrtgpu_batch* b = ws.b;
  const int32_t nq = r.nq;
  int rc = batch_compile(b, ix, r, st);
  const size_t n = (size_t)nq * n_hits;
  if (!rc) rc = b->sd_docs.upload_async(docs, n, st);
  if (!rc && counts) rc = b->sd_counts.upload_async(counts, (size_t)nq, st);
  if (!rc) rc = launch_score_docs(b, ix, nq, n_hits, counts != nullptr, st);
  if (rc) return rc;
  cudaError_t e = cudaMemcpyAsync(out_matches, b->sd_match.p, n, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(out_scores, b->sd_scores.p, n * sizeof(float), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return NRTGPU_ERR_CUDA; }
  return NRTGPU_OK;
}

// nrtgpu_rescore_query / nrtgpu_rescore_query_tree
static int rescore_query_impl(const char* fn, nrtgpu_index* ix, const BatchRequest& r, int32_t n_hits, const int32_t* counts,
                              int32_t window, double query_weight, double rescore_weight, void* stream, int32_t* docs,
                              float* scores, int32_t* out_counts) {
  if (!ix || !docs || !scores || n_hits <= 0 || window <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": bad argument");
  if (n_hits > kHybCap) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, std::string(fn) + ": more than 4096 hits per query");
  cudaStream_t st = (cudaStream_t)stream;
  WorkspaceLease ws(ix);
  nrtgpu_batch* b = ws.b;
  const int32_t nq = r.nq;
  int rc = batch_compile(b, ix, r, st);
  const size_t n = (size_t)nq * n_hits;
  // Lucene QueryRescorer.rescore(searcher, hits, topN = windowSize): EVERY first-pass hit is combined and the list
  // re-sorted (score desc, doc asc); then the first topN are kept
  std::vector<int32_t> wc((size_t)nq);
  for (int q = 0; q < nq; ++q) {
    wc[(size_t)q] = counts ? counts[q] : n_hits;
    if (wc[(size_t)q] < 0 || wc[(size_t)q] > n_hits) NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": counts out of range");
  }
  if (!rc) rc = b->sd_docs.upload_async(docs, n, st);
  if (!rc) rc = b->sd_first.upload_async(scores, n, st);
  if (!rc) rc = b->sd_counts.upload_async(wc.data(), (size_t)nq, st);
  if (!rc) rc = launch_score_docs(b, ix, nq, n_hits, true, st);
  if (rc) return rc;
  RescoreLaunch P;
  P.nq = nq; P.n_hits = n_hits; P.counts = b->sd_counts.p; P.docs = b->sd_docs.p; P.scores = b->sd_first.p;
  P.second_matches = b->sd_match.p; P.second_scores = b->sd_scores.p; P.query_weight = query_weight; P.rescore_weight = rescore_weight;
  rescore_combine_kernel<<<nq, kHybThreads, 0, st>>>(P);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(docs, b->sd_docs.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(scores, b->sd_first.p, n * sizeof(float), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return NRTGPU_ERR_CUDA; }
  if (out_counts) for (int q = 0; q < nq; ++q) out_counts[q] = std::min(wc[(size_t)q], window);
  return NRTGPU_OK;
}

int nrtgpu_score_docs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                      const nrtgpu_query* queries, int32_t nq, int32_t n_hits, const int32_t* docs,
                      const int32_t* counts, void* stream, uint8_t* out_matches, float* out_scores) {
  return score_docs_impl("nrtgpu_score_docs", ix, compile_only_request(clauses, n_clauses, queries, nq), n_hits, docs, counts, stream,
                         out_matches, out_scores);
}

int nrtgpu_rescore_query(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t n_hits, const int32_t* counts,
                         int32_t window, double query_weight, double rescore_weight, void* stream,
                         int32_t* docs, float* scores, int32_t* out_counts) {
  return rescore_query_impl("nrtgpu_rescore_query", ix, compile_only_request(clauses, n_clauses, queries, nq), n_hits, counts, window,
                            query_weight, rescore_weight, stream, docs, scores, out_counts);
}

// the compile-only request of the tree entry points: that of nrtgpu_score_docs with the node and phrase tables
static int compile_only_tree_request(BatchRequest* r, const nrtgpu_node* nodes, int32_t n_nodes, const nrtgpu_phrase* phrases,
                                     int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms) {
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  if (n_nodes > 0) { r->nodes = nodes; r->n_nodes = n_nodes; }
  return phrase_request(r, phrases, n_phrases, phrase_terms, n_phrase_terms);
}

int nrtgpu_score_docs_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                           int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                           const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                           int32_t nq, int32_t n_hits, const int32_t* docs, const int32_t* counts, void* stream,
                           uint8_t* out_matches, float* out_scores) {
  BatchRequest r = compile_only_request(clauses, n_clauses, queries, nq);
  int rc = compile_only_tree_request(&r, nodes, n_nodes, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc) return rc;
  return score_docs_impl("nrtgpu_score_docs_tree", ix, r, n_hits, docs, counts, stream, out_matches, out_scores);
}

int nrtgpu_rescore_query_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                              int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                              const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                              int32_t nq, int32_t n_hits, const int32_t* counts, int32_t window, double query_weight,
                              double rescore_weight, void* stream, int32_t* docs, float* scores, int32_t* out_counts) {
  BatchRequest r = compile_only_request(clauses, n_clauses, queries, nq);
  int rc = compile_only_tree_request(&r, nodes, n_nodes, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc) return rc;
  return rescore_query_impl("nrtgpu_rescore_query_tree", ix, r, n_hits, counts, window, query_weight, rescore_weight, stream, docs,
                            scores, out_counts);
}

int nrtgpu_fetch_columns(nrtgpu_index* ix, const int32_t* col_ids, int32_t n_cols, const int32_t* docs, int32_t n,
                         void* stream, int64_t* out_values, uint8_t* out_has) {
  if (!ix || !col_ids || !docs || !out_values || !out_has || n_cols <= 0 || n <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_fetch_columns: bad argument");
  for (int i = 0; i < n_cols; ++i) if (col_ids[i] < 0 || col_ids[i] >= ix->n_columns) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_fetch_columns: column out of range");
  for (int i = 0; i < n_cols; ++i) if (ix->col_multi[(size_t)col_ids[i]]) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nrtgpu_fetch_columns: multi-valued column");
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> g(ix->fetch_mu);
  int rc;
  const size_t total = (size_t)n_cols * (size_t)n;
  if ((rc = ix->f_cols.upload_async(col_ids, (size_t)n_cols, st)) || (rc = ix->f_docs.upload_async(docs, (size_t)n, st)) ||
      (rc = ix->f_vals.alloc(total)) || (rc = ix->f_has.alloc(total))) return rc;
  FetchLaunch F; F.ix = ix->view(); F.col_ids = ix->f_cols.p; F.n_cols = n_cols; F.docs = ix->f_docs.p; F.n = n;
  F.out_values = ix->f_vals.p; F.out_has = ix->f_has.p;
  fetch_columns_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(F);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpyAsync(out_values, ix->f_vals.p, total * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out_has, ix->f_has.p, total, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  return NRTGPU_OK;
}

int nrtgpu_search_bool_packed(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                              const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                              const nrtgpu_search_limits* limits, void* stream, int32_t* d_record) {
  if (!d_record) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_bool_packed: NULL record");
  SearchOut o; o.d_record = d_record;
  return search_bool_impl(ix, BatchRequest{clauses, n_clauses, queries, nq, top_k, total_hits_threshold, flags}, limits, stream, o);
}

int nrtgpu_merge_topk_device(nrtgpu_ctx* ctx, int32_t n_lists, int32_t nq, int32_t top_k,
                             const int32_t* d_docs, const float* d_scores, const int32_t* d_counts,
                             int32_t* d_out_docs, float* d_out_scores, int32_t* d_out_counts, void* stream) {
  if (!ctx || n_lists <= 0 || nq <= 0 || top_k <= 0 || top_k > kMaxTopK) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_merge_topk_device: bad argument");
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  MergePairsLaunch M;
  M.docs = d_docs; M.scores = d_scores; M.counts = d_counts; M.n_lists = n_lists; M.top_k = top_k; M.nq = nq;
  M.stride_hits = (int64_t)nq * top_k; M.stride_counts = nq;
  M.out_docs = d_out_docs; M.out_scores = d_out_scores; M.out_counts = d_out_counts;
  M.totals = nullptr; M.flags = nullptr; M.stride_totals = 0; M.stride_flags = 0; M.out_total = nullptr; M.out_flags = nullptr;
  merge_pairs_kernel<<<nq, kMergeThreads, 0, (cudaStream_t)stream>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// A kNN boost is a BoostQuery boost: finite and not negative (Lucene's BoostQuery constructor refuses anything else, -0
// included). The rank-safety certificate depends on it: score * boost must not decrease when the score grows, or the
// candidate stage keeps the worst vectors and knn_score_upper_bound certifies them.
static bool knn_boosts_valid(const float* boosts, int32_t nq) {
  for (int32_t q = 0; boosts && q < nq; ++q) if (!std::isfinite(boosts[q]) || std::signbit(boosts[q])) return false;
  return true;
}

// nrtgpu_search_knn and nrtgpu_search_knn_timed once their arguments are checked
static int knn_search_checked(nrtgpu_index* ix, const KnnRequest& req, void* stream, const KnnPages& out, float* stage_ms) {
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  std::lock_guard<std::mutex> g(ix->knn_mu);
  return knn_search_host(ix->knn_corpus(), req, ix->knn_scratch, (cudaStream_t)stream, out, stage_ms, &ix->knn_last_uncertified);
}

int nrtgpu_search_knn(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k, const float* boosts,
                      const uint8_t* filter, void* stream, int32_t* out_docs, float* out_scores,
                      int32_t* out_counts) {
  if (!ix || !queries || !out_docs || !out_scores || !out_counts) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn: NULL argument");
  if (ix->vec_dims <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn: index has no vector field");
  if (nq <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn: nq must be > 0");
  if (k <= 0 || k > kMaxTopK) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn: k out of range");
  if (!knn_boosts_valid(boosts, nq)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn: a boost must be finite and >= 0");
  return knn_search_checked(ix, KnnRequest{queries, nq, k, boosts, filter, nullptr, nullptr, 0}, stream,
                            KnnPages{out_docs, out_scores, out_counts}, nullptr);
}

int nrtgpu_search_knn_timed(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k, void* stream, int32_t* out_docs,
                            float* out_scores, int32_t* out_counts, float* stage_ms /*[3]: gemm, select, rescore*/) {
  if (!ix || !queries || !out_docs || !out_scores || !out_counts || !stage_ms) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_timed: NULL argument");
  if (ix->vec_dims <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_timed: index has no vector field");
  if (nq <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_timed: nq must be > 0");
  if (k <= 0 || k > kMaxTopK / 4) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_timed: k out of range");
  return knn_search_checked(ix, KnnRequest{queries, nq, k, nullptr, nullptr, nullptr, nullptr, 0}, stream,
                            KnnPages{out_docs, out_scores, out_counts}, stage_ms);
}

int32_t nrtgpu_knn_last_uncertified(const nrtgpu_index* ix) { return ix ? ix->knn_last_uncertified : 0; }

struct KnnFilterRows { const uint32_t* bits = nullptr; int32_t* ord_cnt = nullptr; std::vector<int32_t> cnt; };

// The rows of the filters row_filter[] of b (the compiled filter queries): bit d of row r of `rows` (the caller's device
// buffer, [n_rows][words]) is set iff live doc d matches filter row_filter[r]; cnt[r] counts them, ord_cnt (device [n_rows],
// zeroed) is the kNN gather path's. The term bitmaps and row metadata live in the caller's scratch sc. Asynchronous on st:
// the caller synchronises it before it reads cnt.
static int filter_rows(nrtgpu_index* ix, const nrtgpu_batch* b, const std::vector<int32_t>& row_filter, KnnScratch& sc,
                       uint32_t* dRows, cudaStream_t st, KnnFilterRows& out) {
  const int n_rows = (int)row_filter.size(), words = (ix->n_docs + 31) / 32;
  // ---- group the rows so that the bitmaps of a group's distinct terms fit kKnnFilterTermBytes; a term clause points
  //      at its term's bitmap inside its group (terms without postings at none)
  const int n_cl = (int)b->cb.clauses.size();
  std::vector<int32_t> clause_term((size_t)std::max(n_cl, 1), -1);
  std::vector<int64_t> term_base, term_pre(1, 0);
  std::vector<int> grp_row{0}, grp_term{0};   // group g: rows [grp_row[g], grp_row[g + 1]), terms [grp_term[g], grp_term[g + 1])
  std::unordered_map<int64_t, int> group_terms;   // post_base -> term index in the current group
  const size_t term_bytes = (size_t)words * 4;
  for (int r = 0; r < n_rows; ++r) {
    const DevQuery& q = b->cb.queries[(size_t)row_filter[(size_t)r]];
    int fresh = 0;
    for (int i = 0; i < q.n_clauses; ++i) {
      const DevClause& c = b->cb.clauses[(size_t)q.clause_begin + i];
      if (c.kind == NRTGPU_TERM && c.n_post > 0 && !group_terms.count(c.post_base)) ++fresh;
    }
    const int rows_in = r - grp_row.back();
    if (rows_in > 0 && (rows_in == 65535 || (group_terms.size() + fresh) * term_bytes > kKnnFilterTermBytes)) {
      grp_row.push_back(r); grp_term.push_back((int)term_base.size()); group_terms.clear();
    }
    for (int i = 0; i < q.n_clauses; ++i) {
      const int ci = q.clause_begin + i;
      const DevClause& c = b->cb.clauses[(size_t)ci];
      if (c.kind != NRTGPU_TERM || c.n_post == 0) continue;
      const auto [it, added] = group_terms.emplace(c.post_base, (int)group_terms.size());
      if (added) { term_base.push_back(c.post_base); term_pre.push_back(term_pre.back() + c.n_post); }
      clause_term[(size_t)ci] = it->second;
    }
  }
  grp_row.push_back(n_rows); grp_term.push_back((int)term_base.size());
  const int n_terms = (int)term_base.size();
  int64_t* dTerm = nullptr; int32_t* dMeta = nullptr;
  NRT_KNN_GET(KnnSlot::Terms, dTerm, (size_t)(2 * n_terms + 1) * 8);
  NRT_KNN_GET(KnnSlot::RowMeta, dMeta, (size_t)(3 * n_rows + n_cl + 1) * 4);   // row_filter | row_cnt | ord_cnt | clause_term
  int32_t *dRowFilter = dMeta, *dRowCnt = dMeta + n_rows, *dClauseTerm = dMeta + 3 * n_rows;
  if (n_terms) NRT_CUDA_TRY(cudaMemcpyAsync(dTerm, term_base.data(), (size_t)n_terms * 8, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(dTerm + n_terms, term_pre.data(), (size_t)(n_terms + 1) * 8, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(dRowFilter, row_filter.data(), (size_t)n_rows * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemsetAsync(dRowCnt, 0, (size_t)2 * n_rows * 4, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(dClauseTerm, clause_term.data(), clause_term.size() * 4, cudaMemcpyHostToDevice, st));
  // ---- per group: term bitmaps, then the rows
  size_t group_bytes = 0;
  for (size_t g = 0; g + 1 < grp_row.size(); ++g) group_bytes = std::max(group_bytes, (size_t)(grp_term[g + 1] - grp_term[g]) * term_bytes);
  uint32_t* dTbits = nullptr;
  NRT_KNN_GET(KnnSlot::TermBits, dTbits, std::max<size_t>(group_bytes, 4));
  for (size_t g = 0; g + 1 < grp_row.size(); ++g) {
    const int t0 = grp_term[g], nt = grp_term[g + 1] - t0;
    if (nt > 0) {
      NRT_CUDA_TRY(cudaMemsetAsync(dTbits, 0, (size_t)nt * term_bytes, st));
      KnnTermScatterLaunch S; S.post_docs = ix->post_docs.p; S.term_base = dTerm + t0; S.term_pre = dTerm + n_terms + t0;
      S.n_terms = nt; S.words = words; S.tbits = dTbits;
      const int64_t posts = term_pre[(size_t)t0 + nt] - term_pre[(size_t)t0];
      knn_term_scatter_kernel<<<(unsigned)std::min<int64_t>((posts + 255) / 256, 8 * 1024), 256, 0, st>>>(S);
      NRT_CUDA_TRY(cudaGetLastError());
    }
    KnnFilterRowsLaunch R; R.ix = ix->view(); R.clauses = b->clauses.p; R.filters = b->queries.p; R.row_filter = dRowFilter;
    R.clause_term = dClauseTerm; R.tbits = dTbits; R.row0 = grp_row[g]; R.words = words; R.rows = dRows; R.row_cnt = dRowCnt;
    knn_filter_rows_kernel<<<dim3((unsigned)((words + 255) / 256), (unsigned)(grp_row[g + 1] - grp_row[g])), 256, 0, st>>>(R);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  out.bits = dRows; out.ord_cnt = dMeta + 2 * n_rows; out.cnt.assign((size_t)n_rows, 0);
  NRT_CUDA_TRY(cudaMemcpyAsync(out.cnt.data(), dRowCnt, (size_t)n_rows * 4, cudaMemcpyDeviceToHost, st));
  return NRTGPU_OK;
}

// The rows of a kNN call's filters (filter_rows in the index's kNN scratch); adds their device time to the filter statistics.
static int knn_filter_rows(nrtgpu_index* ix, const nrtgpu_batch* b, const std::vector<int32_t>& row_filter, cudaStream_t st,
                           KnnFilterRows& out) {
  KnnScratch& sc = ix->knn_scratch;
  uint32_t* dRows = nullptr;
  NRT_KNN_GET(KnnSlot::Rows, dRows, row_filter.size() * (size_t)((ix->n_docs + 31) / 32) * 4);
  if (!ix->knn_ev[0]) for (auto& e : ix->knn_ev) NRT_CUDA_TRY(cudaEventCreate(&e));
  NRT_CUDA_TRY(cudaEventRecord(ix->knn_ev[0], st));
  if (int rc = filter_rows(ix, b, row_filter, sc, dRows, st, out)) return rc;
  NRT_CUDA_TRY(cudaEventRecord(ix->knn_ev[1], st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  float ms = 0.0f;
  NRT_CUDA_TRY(cudaEventElapsedTime(&ms, ix->knn_ev[0], ix->knn_ev[1]));
  ix->knn_last_filter_ms += ms;
  return NRTGPU_OK;
}

// The rows of the batch's FILTER aggregations on its image (batch_build; nothing without them): the k-th FILTER aggregation
// owns row k of agg_rows, the filter queries' rows first (filter_rows on the filters compiled into agg_fq, as the kNN
// filters are), then the value sets' (agg_value_set_kernel, each set sorted and de-duplicated here). A filter under a filter
// then ANDs its parent's row into its own, in request order, so one row gates each aggregation: agg_gate[i] is aggregation
// i's own row for a FILTER aggregation, its filter_agg's row for a TERMS one (batch_agg_codes turns them into codes).
static int batch_filter_rows(nrtgpu_batch* b, const BatchRequest& r, cudaStream_t st) {
  std::fill(b->agg_gate, b->agg_gate + kMaxAggs, nullptr);
  const CompiledBatch& cb = b->cb;
  nrtgpu_index* ix = b->ix;
  std::vector<int32_t> row_filter, sets, row_of(cb.aggs.size(), -1);
  for (size_t i = 0; i < cb.aggs.size(); ++i)
    if (cb.aggs[i].kind == NRTGPU_AGG_FILTER) {
      if (cb.agg_filters[i].kind == NRTGPU_AGG_FILTER_QUERY) { row_of[i] = (int32_t)row_filter.size(); row_filter.push_back(cb.agg_filters[i].query); }
      else sets.push_back((int32_t)i);
    }
  const int n_rows = (int)(row_filter.size() + sets.size()), words = (ix->n_docs + 31) / 32;
  if (n_rows == 0) return NRTGPU_OK;
  int rc;
  if (cb.agg_filter_queries) {   // compiled here, before any run, so that a refused filter writes no output
    if (!b->agg_fq) b->agg_fq.reset(new nrtgpu_batch);
    if ((rc = batch_compile(b->agg_fq.get(), ix, compile_only_request(r.filter_clauses, r.n_filter_clauses, r.filter_queries,
                                                                      r.n_filter_queries), st))) return rc;
  }
  if (words == 0) return NRTGPU_OK;   // an image without docs: nothing is collected
  if ((rc = b->agg_rows.alloc((size_t)n_rows * words))) return rc;
  KnnFilterRows qrows;
  if (!row_filter.empty() && (rc = filter_rows(ix, b->agg_fq.get(), row_filter, b->agg_scratch, b->agg_rows.p, st, qrows))) return rc;
  std::vector<int64_t> vals;   // the sets, sorted and distinct, one after the other
  std::vector<size_t> set_at;
  for (int32_t i : sets) {
    const nrtgpu_agg_filter& f = cb.agg_filters[(size_t)i];
    set_at.push_back(vals.size());
    const size_t at = vals.size();
    vals.insert(vals.end(), f.values, f.values + f.n_values);
    std::sort(vals.begin() + (std::ptrdiff_t)at, vals.end());
    vals.erase(std::unique(vals.begin() + (std::ptrdiff_t)at, vals.end()), vals.end());
  }
  set_at.push_back(vals.size());
  if ((rc = b->agg_set.upload_async(vals.data(), vals.size(), st))) return rc;
  for (size_t k = 0; k < sets.size(); ++k) {
    const int32_t i = sets[k];
    row_of[(size_t)i] = (int32_t)(row_filter.size() + k);
    AggValueSetLaunch L;
    L.ix = ix->view(); L.column = cb.agg_filters[(size_t)i].column; L.n_set = (int32_t)(set_at[k + 1] - set_at[k]); L.words = words;
    L.keyword = cb.agg_filters[(size_t)i].kind == NRTGPU_AGG_FILTER_KEYWORD_SET;
    L.set = b->agg_set.p + set_at[k]; L.row = b->agg_rows.p + (size_t)row_of[(size_t)i] * words;
    agg_value_set_kernel<<<(unsigned)(((int64_t)words * 32 + 255) / 256), 256, 0, st>>>(L);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  for (size_t i = 0; i < cb.aggs.size(); ++i) {
    const nrtgpu_aggregation& a = cb.aggs[i];
    uint32_t* own = row_of[i] >= 0 ? b->agg_rows.p + (size_t)row_of[i] * words : nullptr;
    const uint32_t* parent = a.filter_agg > 0 ? b->agg_gate[a.filter_agg - 1] : nullptr;
    if (own && parent) {
      row_and_kernel<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(own, parent, words);
      NRT_CUDA_TRY(cudaGetLastError());
    }
    b->agg_gate[i] = own ? own : parent;
  }
  NRT_CUDA_TRY(cudaStreamSynchronize(st));   // (the host sets and counts are read by the async copies)
  return NRTGPU_OK;
}

// Gather path of the queries first .. g.nq - 1 of g: each of their rows' ordinals listed once, then scored exactly.
static int knn_gather_host(const KnnCorpus& corpus, const KnnRequest& g, int first, const KnnFilterRows& rows, KnnScratch& sc,
                           cudaStream_t st, const KnnPages& out) {
  const int nq = g.nq, dims = corpus.dims, n_vec = corpus.n, n_rows = (int)rows.cnt.size();
  std::vector<int32_t> gsel, grows;
  std::vector<int64_t> ord_begin((size_t)n_rows, -1);   // -1: no query of the gather path has the row
  int64_t total = 0; int max_cnt = 0;
  for (int q = first; q < nq; ++q) {
    const int r = g.qrow[q];
    gsel.push_back(q);
    if (ord_begin[(size_t)r] >= 0) continue;
    grows.push_back(r);
    ord_begin[(size_t)r] = total; total += rows.cnt[(size_t)r]; max_cnt = std::max(max_cnt, rows.cnt[(size_t)r]);
  }
  int32_t *dOrds = nullptr, *dGrows = nullptr, *dQrow = nullptr; int64_t* dOrdBegin = nullptr; float *dQ = nullptr, *dB = nullptr;
  NRT_KNN_GET(KnnSlot::GatherQ, dQ, (size_t)nq * dims * 4);
  NRT_KNN_GET(KnnSlot::Ords, dOrds, (size_t)std::max<int64_t>(total, 1) * 4);
  NRT_KNN_GET(KnnSlot::OrdBegin, dOrdBegin, (size_t)n_rows * 8);
  NRT_KNN_GET(KnnSlot::GatherRows, dGrows, grows.size() * 4);
  NRT_KNN_GET(KnnSlot::GatherQrow, dQrow, (size_t)nq * 4);
  NRT_CUDA_TRY(cudaMemcpyAsync(dQ, g.queries, (size_t)nq * dims * 4, cudaMemcpyHostToDevice, st));
  if (g.boosts) { NRT_KNN_GET(KnnSlot::GatherBoosts, dB, (size_t)nq * 4); NRT_CUDA_TRY(cudaMemcpyAsync(dB, g.boosts, (size_t)nq * 4, cudaMemcpyHostToDevice, st)); }
  NRT_CUDA_TRY(cudaMemcpyAsync(dOrdBegin, ord_begin.data(), (size_t)n_rows * 8, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(dGrows, grows.data(), grows.size() * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(dQrow, g.qrow, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
  KnnFilterOrdsLaunch O; O.rows = rows.bits; O.words = g.words; O.ord_begin = dOrdBegin; O.vec_docs = corpus.vec_docs; O.n_vec = n_vec;
  O.ords = dOrds; O.ord_cnt = rows.ord_cnt;
  const int items = corpus.vec_docs ? n_vec : (n_vec + 31) / 32;
  for (size_t g0 = 0; g0 < grows.size(); g0 += 65535) {
    O.grows = dGrows + g0;
    knn_filter_ords_kernel<<<dim3((unsigned)((items + 255) / 256), (unsigned)std::min<size_t>(65535, grows.size() - g0)), 256, 0, st>>>(O);
    NRT_CUDA_TRY(cudaGetLastError());
  }
  KnnExactLaunch X; X.Q = dQ; X.boosts = dB; X.filter = nullptr; X.k = g.k; X.qfilter = rows.bits; X.qrow = dQrow; X.qwords = g.words;
  X.ords = dOrds; X.ord_begin = dOrdBegin; X.ord_cnt = rows.ord_cnt;
  return knn_exact_host(corpus, sc, st, X, std::max(1, (max_cnt + kKnnExactChunk - 1) / kKnnExactChunk), gsel, out);
}

// Filtered kNN of the queries whose row req.qrow[q] is in [r0, r1) (r0 = 0: also those without a filter). A query whose
// filter matches at most n_vec / kKnnGatherRatio docs is scored over those docs only, every other one by the candidate
// stage with its row, on a prefix of the batch packed with those first. Caller holds ix->knn_mu.
static int knn_filtered_group(nrtgpu_index* ix, const nrtgpu_batch* b, const KnnRequest& req,
                              const std::vector<int32_t>& row_filter, int r0, int r1, cudaStream_t st, const KnnPages& out) {
  KnnFilterRows rows;
  if (r1 > r0) if (int rc = knn_filter_rows(ix, b, {row_filter.begin() + r0, row_filter.begin() + r1}, st, rows)) return rc;
  const KnnCorpus corpus = ix->knn_corpus();
  const bool can_gather = !corpus.vec_docs || ix->vec_docs_ascending;
  std::vector<int32_t> lrow((size_t)req.nq, -1), order, gsel;   // lrow: row in this group (-1: none)
  for (int q = 0; q < req.nq; ++q) {
    const int r = req.qrow[q], lr = r < 0 ? -1 : r - r0;
    if (r >= 0 ? r >= r1 || lr < 0 : r0 > 0) continue;
    lrow[(size_t)q] = lr;
    (lr >= 0 && can_gather && (int64_t)rows.cnt[(size_t)lr] * kKnnGatherRatio <= (int64_t)corpus.n ? gsel : order).push_back(q);
  }
  ix->knn_last_gather += (int32_t)gsel.size();
  const int nt = (int)order.size();
  order.insert(order.end(), gsel.begin(), gsel.end());
  KnnRequest greq = req; greq.qrow = r1 > r0 ? lrow.data() : nullptr; greq.d_rows = rows.bits; greq.words = (ix->n_docs + 31) / 32;
  return knn_run_subset(greq, corpus.dims, order, out, [&](const KnnRequest& g, const KnnPages& o) {
    KnnRequest t = g; t.nq = nt; int32_t unc = 0;
    if (int rc = nt > 0 ? knn_search_host(corpus, t, ix->knn_scratch, st, o, nullptr, &unc) : NRTGPU_OK) return rc;
    ix->knn_last_uncertified += unc;
    return g.nq > nt ? knn_gather_host(corpus, g, nt, rows, ix->knn_scratch, st, o) : NRTGPU_OK;
  });
}

int nrtgpu_search_knn_filtered(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k, const float* boosts,
                               const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                               const nrtgpu_query* filters, int32_t n_filters, const int32_t* filter_of,
                               void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts) {
  if (!ix || !queries || !filter_of || !out_docs || !out_scores || !out_counts || (n_filters > 0 && !filters))
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: NULL argument");
  if (nq <= 0 || n_filters < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: nq must be > 0 and n_filters >= 0");
  if (ix->vec_dims <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: index has no vector field");
  if (k <= 0 || k > kMaxTopK) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: k out of range");
  if (!knn_boosts_valid(boosts, nq)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: a boost must be finite and >= 0");
  for (int f = 0; f < n_filters; ++f)
    if (filters[f].has_after) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: a filter query has no searchAfter");
  // rows: the filters some query uses, in order of first use
  std::vector<int32_t> row_of((size_t)n_filters, -1), row_filter, qrow((size_t)nq, -1);
  for (int q = 0; q < nq; ++q) {
    const int f = filter_of[q];
    if (f < -1 || f >= n_filters) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_knn_filtered: filter_of out of range");
    if (f < 0) continue;
    if (row_of[(size_t)f] < 0) { row_of[(size_t)f] = (int32_t)row_filter.size(); row_filter.push_back(f); }
    qrow[(size_t)q] = row_of[(size_t)f];
  }
  NRT_CUDA_TRY(cudaSetDevice(ix->ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::optional<WorkspaceLease> ws;
  nrtgpu_batch* b = nullptr;
  int rc = NRTGPU_OK;
  if (n_filters > 0) {   // the filters compile as a batch of flat BooleanQuerys (clause checks, UNSUPPORTED shapes)
    b = ws.emplace(ix).b;
    rc = batch_compile(b, ix, compile_only_request(filter_clauses, n_filter_clauses, filters, n_filters), st);
  }
  if (!rc) {
    std::lock_guard<std::mutex> g(ix->knn_mu);
    ix->knn_last_gather = 0; ix->knn_last_uncertified = 0; ix->knn_last_filter_ms = 0.0f;
    // bounded scratch: the queries run in groups whose distinct rows fit kKnnFilterRowBytes. Rows are numbered in order of
    // first use, so group g owns rows [g * per, (g + 1) * per); a query goes with its row (no filter: group 0).
    const int n_rows = (int)row_filter.size();
    const int per = (int)std::max<int64_t>(1, std::min<int64_t>(65535, (int64_t)kKnnFilterRowBytes / ((ix->n_docs + 31) / 32 * 4)));
    const KnnRequest req{queries, nq, k, boosts, nullptr, nullptr, qrow.data(), 0};
    for (int r0 = 0; !rc && (r0 == 0 || r0 < n_rows); r0 += per)
      rc = knn_filtered_group(ix, b, req, row_filter, r0, std::min(n_rows, r0 + per), st, KnnPages{out_docs, out_scores, out_counts});
  }
  return rc;
}

int nrtgpu_knn_filter_stats(const nrtgpu_index* ix, int32_t* out_gather_queries, float* out_filter_ms) {
  if (!ix) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_knn_filter_stats: NULL index");
  if (out_gather_queries) *out_gather_queries = ix->knn_last_gather;
  if (out_filter_ms) *out_filter_ms = ix->knn_last_filter_ms;
  return NRTGPU_OK;
}

// weighted RRF (mode 0) or score-order (MAX / SUM / AVG) blend of R retrievers' lists; HOST buffers, pooled device scratch
static int blend_impl(nrtgpu_ctx* ctx, int32_t mode, int32_t R, int32_t nq, int32_t top_in, const int32_t* docs, const float* scores,
                      const int32_t* counts, const float* boosts, int32_t rank_constant, int32_t top_out, int32_t* out_docs,
                      float* out_scores, int32_t* out_counts, int32_t* out_total) {
  if (!ctx || !docs || !counts || !boosts || !out_docs || !out_scores || !out_counts || !out_total || (mode != 0 && !scores))
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_blend: NULL argument");
  if (R <= 0 || nq <= 0 || top_in <= 0 || top_out <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_blend: sizes must be > 0");
  if ((int64_t)R * top_in > kHybCap || top_in > 65535 || R > 65535) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nrtgpu_blend: more than 4096 hits per query");
  for (int64_t i = 0; i < (int64_t)R * nq; ++i)
    if (counts[i] < 0 || counts[i] > top_in) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_blend: counts[] outside [0, top_in]");
  // WeightedRrfBlenderOperation.java:47-49: rankConstant <= 0 selects DEFAULT_K = 60
  const int k = rank_constant > 0 ? rank_constant : 60;
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  const size_t nd = (size_t)R * nq * top_in, nc = (size_t)R * nq, no = (size_t)nq * top_out;
  std::lock_guard<std::mutex> g(ctx->hyb_mu);
  int rc;
  // one pooled allocation, carved up (all parts 4-byte types)
  const size_t words = nd * 2 + nc + (size_t)R + no * 2 + (size_t)nq * 2;
  if ((rc = ctx->hyb_scratch.alloc(words))) return rc;
  int32_t* p = ctx->hyb_scratch.p;
  int32_t* d_docs = p; p += nd;
  float* d_scores = (float*)p; p += nd;
  int32_t* d_counts = p; p += nc;
  float* d_boosts = (float*)p; p += R;
  int32_t* d_od = p; p += no;
  float* d_os = (float*)p; p += no;
  int32_t* d_oc = p; p += nq;
  int32_t* d_ot = p;
  cudaStream_t st = 0;
  NRT_CUDA_TRY(cudaMemcpyAsync(d_docs, docs, nd * 4, cudaMemcpyHostToDevice, st));
  if (mode != 0) NRT_CUDA_TRY(cudaMemcpyAsync(d_scores, scores, nd * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_counts, counts, nc * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_boosts, boosts, (size_t)R * 4, cudaMemcpyHostToDevice, st));
  RrfLaunch P;
  P.docs = d_docs; P.counts = d_counts; P.boosts = d_boosts; P.scores = mode != 0 ? d_scores : nullptr; P.mode = mode;
  P.R = R; P.nq = nq; P.top_in = top_in; P.rank_constant = k; P.top_out = top_out;
  P.out_docs = d_od; P.out_scores = d_os; P.out_counts = d_oc; P.out_total = d_ot;
  rrf_blend_kernel<<<nq, kHybThreads, 0, st>>>(P);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpyAsync(out_docs, d_od, no * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out_scores, d_os, no * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out_counts, d_oc, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out_total, d_ot, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  return NRTGPU_OK;
}

int nrtgpu_blend_rrf(nrtgpu_ctx* ctx, int32_t R, int32_t nq, int32_t top_in, const int32_t* docs, const int32_t* counts,
                     const float* boosts, int32_t rank_constant, int32_t top_out, int32_t* out_docs, float* out_scores,
                     int32_t* out_counts, int32_t* out_total) {
  return blend_impl(ctx, 0, R, nq, top_in, docs, nullptr, counts, boosts, rank_constant, top_out, out_docs, out_scores, out_counts, out_total);
}

int nrtgpu_blend_scores(nrtgpu_ctx* ctx, int32_t score_mode, int32_t R, int32_t nq, int32_t top_in, const int32_t* docs,
                        const float* scores, const int32_t* counts, const float* boosts, int32_t top_out, int32_t* out_docs,
                        float* out_scores, int32_t* out_counts, int32_t* out_total) {
  if (score_mode < NRTGPU_BLEND_MAX || score_mode > NRTGPU_BLEND_AVG) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_blend_scores: bad score mode");
  return blend_impl(ctx, score_mode, R, nq, top_in, docs, scores, counts, boosts, 0, top_out, out_docs, out_scores, out_counts, out_total);
}

int nrtgpu_rescore_combine(nrtgpu_ctx* ctx, int32_t nq, int32_t n_hits, const int32_t* counts, int32_t* docs, float* scores,
                           const uint8_t* second_matches, const float* second_scores, double query_weight,
                           double rescore_weight) {
  if (!ctx || !docs || !scores || !second_matches || !second_scores) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_rescore_combine: NULL argument");
  if (nq <= 0 || n_hits <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_rescore_combine: sizes must be > 0");
  if (n_hits > kHybCap) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nrtgpu_rescore_combine: more than 4096 hits per query");
  if (counts) for (int q = 0; q < nq; ++q) if (counts[q] < 0 || counts[q] > n_hits) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_rescore_combine: counts[] outside [0, n_hits]");
  NRT_CUDA_TRY(cudaSetDevice(ctx->device));
  const size_t n = (size_t)nq * n_hits;
  std::lock_guard<std::mutex> g(ctx->hyb_mu);
  int rc;
  if ((rc = ctx->hyb_scratch.alloc(n * 3 + (n + 3) / 4 + (size_t)nq))) return rc;
  int32_t* p = ctx->hyb_scratch.p;
  int32_t* d_docs = p; p += n;
  float* d_scores = (float*)p; p += n;
  float* d_second = (float*)p; p += n;
  int32_t* d_counts = p; p += nq;
  uint8_t* d_match = (uint8_t*)p;
  cudaStream_t st = 0;
  NRT_CUDA_TRY(cudaMemcpyAsync(d_docs, docs, n * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_scores, scores, n * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_match, second_matches, n, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_second, second_scores, n * 4, cudaMemcpyHostToDevice, st));
  if (counts) NRT_CUDA_TRY(cudaMemcpyAsync(d_counts, counts, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
  RescoreLaunch P;
  P.nq = nq; P.n_hits = n_hits; P.counts = counts ? d_counts : nullptr;
  P.docs = d_docs; P.scores = d_scores; P.second_matches = d_match; P.second_scores = d_second;
  P.query_weight = query_weight; P.rescore_weight = rescore_weight;
  rescore_combine_kernel<<<nq, kHybThreads, 0, st>>>(P);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpyAsync(docs, d_docs, n * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(scores, d_scores, n * 4, cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  return NRTGPU_OK;
}

}  // extern "C"

// ---- searcher over several leaf images of one shard (NRT: a new reader version adds images for the NEW leaves only)
// The reader-wide value dictionary of one column (collect_kernel.cuh, dict_map_kernel): the sorted union of the leaves'
// distinct values, and per leaf the codes that number its docs' values in it. A leaf whose dictionary is the union, or
// which holds no value, counts through its own col_code; every other leaf through a renumbered copy (4 B per doc).
// A keyword column's reader-wide dictionary is the byte-order union of the leaves' term dictionaries, built on the host
// (bytes / off); values stays empty, and a leaf's codes (per doc or per value) are renumbered through its ordinal map,
// which is kept: keyword sorts map the leaf's FieldDoc values to the union through it, and after values back.
struct ReaderDict {
  DevBuf<uint64_t> values;   // [n] ascending, the sortable domain of col_distinct
  int32_t n = 0;
  std::vector<uint8_t> bytes; std::vector<int64_t> off;   // keyword columns: term g of the union is bytes[off[g], off[g + 1])
  std::vector<std::unique_ptr<DevBuf<uint32_t>>> own;   // per leaf: the renumbered codes (unallocated where col_code serves)
  std::vector<const uint32_t*> codes;                   // per leaf: the codes its docs count through
  // keyword columns, per leaf: whether its dictionary is the union, else its ordinal map (leaf term i -> union ordinal,
  // ascending) on the host and on the device (unallocated for a leaf without terms)
  std::vector<uint8_t> same;
  std::vector<std::vector<uint32_t>> hmap;
  std::vector<std::unique_ptr<DevBuf<uint32_t>>> dmap;
};

struct nrtgpu_searcher {
  nrtgpu_ctx* ctx = nullptr;
  std::vector<nrtgpu_index*> leaves;
  std::mutex mu;
  DevBuf<int32_t> records, merged;   // [n_leaves][words], [words]
  std::vector<int32_t> host;
  // per aggregated column, built by its first aggregation and kept for the searcher's life: leaf columns never change
  // (set_live_docs and update_stats leave them alone, and a dictionary keeps the values of deleted docs)
  std::map<int32_t, std::unique_ptr<ReaderDict>> dicts;
  std::map<int32_t, std::unique_ptr<ReaderDict>> kw_dicts;   // the same per keyword column
};

// the reader-wide dictionary of keyword column `column` (built on `st` the first time it is asked for); the caller checked
// that every leaf has the column
static int searcher_kw_dict(nrtgpu_searcher* s, int32_t column, cudaStream_t st, const ReaderDict** out) {
  auto it = s->kw_dicts.find(column);
  if (it != s->kw_dicts.end()) { *out = it->second.get(); return NRTGPU_OK; }
  std::unique_ptr<ReaderDict> d(new ReaderDict);
  auto term = [](const KeywordColumn& c, int32_t t) {
    return std::string(reinterpret_cast<const char*>(c.bytes.data()) + c.off[(size_t)t], (size_t)(c.off[(size_t)t + 1] - c.off[(size_t)t]));
  };
  std::vector<std::string> uni;   // std::string compares as unsigned bytes, then length: BytesRef order
  for (const nrtgpu_index* ix : s->leaves) {
    const KeywordColumn& c = *ix->kw[(size_t)column];
    for (int32_t t = 0; t < c.n_terms; ++t) uni.push_back(term(c, t));
  }
  std::sort(uni.begin(), uni.end());
  uni.erase(std::unique(uni.begin(), uni.end()), uni.end());
  if (uni.size() > (size_t)INT32_MAX / 2) NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "keyword terms: more than 2^30 terms over the leaves");
  d->n = (int32_t)uni.size();
  d->off.assign(1, 0);
  for (const std::string& x : uni) { d->bytes.insert(d->bytes.end(), x.begin(), x.end()); d->off.push_back((int64_t)d->bytes.size()); }
  int rc;
  for (const nrtgpu_index* ix : s->leaves) {
    const KeywordColumn& c = *ix->kw[(size_t)column];
    d->own.emplace_back(new DevBuf<uint32_t>);
    d->dmap.emplace_back(new DevBuf<uint32_t>);
    d->hmap.emplace_back();
    d->same.push_back(c.n_terms == d->n ? 1 : 0);
    const int64_t n_codes = c.n_values;
    if (c.n_terms == d->n || c.n_terms == 0) { d->codes.push_back(c.codes.p); continue; }   // already reader-wide, or all 0
    std::vector<uint32_t>& m = d->hmap.back();
    m.resize((size_t)c.n_terms);
    for (int32_t t = 0; t < c.n_terms; ++t) m[(size_t)t] = (uint32_t)(std::lower_bound(uni.begin(), uni.end(), term(c, t)) - uni.begin());
    DevBuf<uint32_t>& map = *d->dmap.back();
    if ((rc = map.upload_async(m.data(), m.size(), st))) return rc;
    if (n_codes == 0) { d->codes.push_back(c.codes.p); continue; }
    DevBuf<uint32_t>& own = *d->own.back();
    if ((rc = own.alloc((size_t)n_codes))) return rc;
    dict_remap_kernel<<<(unsigned)((n_codes + 255) / 256), 256, 0, st>>>(c.codes.p, n_codes, map.p, own.p);   // (per doc or per value)
    NRT_CUDA_TRY(cudaGetLastError());
    d->codes.push_back(own.p);
  }
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  *out = d.get();
  s->kw_dicts[column] = std::move(d);
  return NRTGPU_OK;
}

// whether every leaf of s has keyword column `column`
static bool searcher_has_kw(const nrtgpu_searcher* s, int32_t column) {
  for (const nrtgpu_index* ix : s->leaves) if (column < 0 || (size_t)column >= ix->kw.size()) return false;
  return true;
}

// The reader-wide dictionaries of the KEYWORD fields of a Sort (orders of the leaves of s, all of that Sort; built on st
// when first asked for): dicts[j] (NULL for the other kinds), and per leaf l maps[l][j], its ordinal map to the union
// (NULL where the leaf's dictionary is the union, or for the other kinds)
static int searcher_sort_kw(nrtgpu_searcher* s, const nrtgpu_sort_order* o, cudaStream_t st, const ReaderDict** dicts,
                            std::vector<std::array<const uint32_t*, kMaxSortFields>>* maps) {
  maps->assign(s->leaves.size(), std::array<const uint32_t*, kMaxSortFields>{});
  for (int j = 0; j < o->n_fields; ++j) {
    dicts[j] = nullptr;
    if (o->spec[j].kind != NRTGPU_SORT_KEYWORD) continue;
    if (int rc = searcher_kw_dict(s, o->spec[j].column, st, &dicts[j])) return rc;
    for (size_t l = 0; l < s->leaves.size(); ++l)
      if (!dicts[j]->same[l]) (*maps)[l][(size_t)j] = dicts[j]->dmap[l]->p;
  }
  return NRTGPU_OK;
}

// a reader-wide KEYWORD code -> the code that leaf l's dictionary gives the same term (the leaf's terms are a subset of
// the union, so its map m is ascending): a held union term 2g + 2 is the leaf's 2i + 2 when m[i] == g, else an odd code;
// the gap 2g + 1 before union term g is the gap before the leaf's first term at or after it
static int64_t kw_code_to_leaf(const ReaderDict& d, size_t l, int64_t c) {
  if (c == 0 || d.same[l]) return c;
  const std::vector<uint32_t>& m = d.hmap[l];
  const uint32_t g = (uint32_t)((c - 1) / 2);
  const size_t i = (size_t)(std::lower_bound(m.begin(), m.end(), g) - m.begin());
  return (c % 2 == 0 && i < m.size() && m[i] == g) ? 2 * (int64_t)i + 2 : 2 * (int64_t)i + 1;
}

// Keyword clauses and keyword value sets of a searcher's request carry reader-wide codes; each leaf receives a copy of
// the clause array (and of the filter records) with its codes mapped by kw_code_to_leaf. That map is monotone and sends a
// union term the leaf lacks to the leaf's gap code beside it, so an inclusive bound keeps exactly the leaf terms that lie
// inside the union bound: for a leaf term with union ordinal u, 2u + 2 >= lo iff its leaf code >= the mapped lo (a lo on
// a held term maps onto that term; one on a missing term or a gap maps onto the gap before the first leaf term above it),
// and symmetrically for hi. The argument is the one behind the sorted after values. A set code maps to the leaf's code of
// the same term, or to an odd code, which matches nothing, where the leaf lacks it. Leaves whose dictionary is the union
// (same[l]) take the caller's arrays.
struct KwLeafRequest {
  const ReaderDict* dict[kMaxAggs] = {};                  // per aggregation: the dictionary of a keyword set
  std::vector<const ReaderDict*> clause_dict, filter_dict;   // per clause / filter clause: a keyword clause's dictionary
  bool any = false;
  std::vector<nrtgpu_clause> clauses, filter_clauses;     // leaf copies
  std::vector<nrtgpu_agg_filter> filters;
  std::vector<std::vector<int64_t>> sets;
};

// the reader-wide dictionaries of the keyword clauses of cl[0 .. n), their columns and codes checked against the union
// with the messages of the single-image call
static int searcher_kw_clauses(nrtgpu_searcher* s, const nrtgpu_clause* cl, int32_t n, cudaStream_t st,
                               std::vector<const ReaderDict*>* dicts, bool* any) {
  dicts->assign((size_t)std::max(n, 0), nullptr);
  for (int32_t i = 0; cl && i < n; ++i) {
    if (cl[i].kind != NRTGPU_KEYWORD_RANGE) continue;
    if (!searcher_has_kw(s, cl[i].id)) NRT_FAIL(NRTGPU_ERR_INVALID, "keyword range: keyword column out of range");
    const ReaderDict* d = nullptr;
    if (int rc = searcher_kw_dict(s, cl[i].id, st, &d)) return rc;
    const int64_t top = 2 * (int64_t)d->n + 1;
    if (cl[i].lo < 1 || cl[i].lo > top || cl[i].hi < 1 || cl[i].hi > top) NRT_FAIL(NRTGPU_ERR_INVALID, "keyword range: keyword code out of range");
    (*dicts)[(size_t)i] = d;
    *any = true;
  }
  return NRTGPU_OK;
}

// the keyword clauses, filter clauses and keyword sets of request r on searcher s (caller holds s->mu)
static int searcher_kw_request(nrtgpu_searcher* s, const BatchRequest& r, cudaStream_t st, KwLeafRequest* k) {
  int rc;
  if ((rc = searcher_kw_clauses(s, r.clauses, r.n_clauses, st, &k->clause_dict, &k->any))) return rc;
  if ((rc = searcher_kw_clauses(s, r.filter_clauses, r.n_filter_clauses, st, &k->filter_dict, &k->any))) return rc;
  for (int i = 0; i < std::min(r.n_aggs, kMaxAggs) && r.agg_filters && r.aggs; ++i) {
    const nrtgpu_agg_filter& f = r.agg_filters[i];
    if (r.aggs[i].kind != NRTGPU_AGG_FILTER || f.kind != NRTGPU_AGG_FILTER_KEYWORD_SET) continue;
    if (!searcher_has_kw(s, f.column)) NRT_FAIL(NRTGPU_ERR_INVALID, "filter aggregation: keyword column out of range");
    if (f.n_values < 0 || (f.n_values > 0 && !f.values)) NRT_FAIL(NRTGPU_ERR_INVALID, "filter aggregation: bad value set");
    if ((rc = searcher_kw_dict(s, f.column, st, &k->dict[i]))) return rc;
    for (int32_t v = 0; v < f.n_values; ++v)
      if (f.values[v] < 1 || f.values[v] > 2 * (int64_t)k->dict[i]->n + 1)
        NRT_FAIL(NRTGPU_ERR_INVALID, "filter aggregation: keyword code out of range");
    k->any = true;
  }
  return NRTGPU_OK;
}

// cl[0 .. n) with the keyword codes of leaf l (dicts from searcher_kw_clauses), in buf, or cl itself when nothing changes
static const nrtgpu_clause* kw_leaf_clauses(const std::vector<const ReaderDict*>& dicts, const nrtgpu_clause* cl, int32_t n, size_t l,
                                            std::vector<nrtgpu_clause>& buf) {
  bool change = false;
  for (int32_t i = 0; i < n; ++i) change |= dicts[(size_t)i] && !dicts[(size_t)i]->same[l];
  if (!change) return cl;
  buf.assign(cl, cl + n);
  for (int32_t i = 0; i < n; ++i)
    if (const ReaderDict* d = dicts[(size_t)i]) { buf[(size_t)i].lo = kw_code_to_leaf(*d, l, cl[i].lo); buf[(size_t)i].hi = kw_code_to_leaf(*d, l, cl[i].hi); }
  return buf.data();
}

// request r as leaf l of the searcher receives it (k from searcher_kw_request)
static BatchRequest kw_leaf_request(KwLeafRequest& k, const BatchRequest& r, size_t l) {
  BatchRequest x = r;
  if (!k.any) return x;
  x.clauses = kw_leaf_clauses(k.clause_dict, r.clauses, r.n_clauses, l, k.clauses);
  x.filter_clauses = kw_leaf_clauses(k.filter_dict, r.filter_clauses, r.n_filter_clauses, l, k.filter_clauses);
  bool sets = false;
  const int n_aggs = std::min(r.n_aggs, kMaxAggs);
  for (int i = 0; i < n_aggs; ++i) sets |= k.dict[i] && !k.dict[i]->same[l];
  if (sets) {
    k.filters.assign(r.agg_filters, r.agg_filters + r.n_aggs);
    k.sets.assign((size_t)n_aggs, {});
    for (int i = 0; i < n_aggs; ++i) {
      if (!k.dict[i]) continue;
      nrtgpu_agg_filter& f = k.filters[(size_t)i];
      for (int32_t v = 0; v < f.n_values; ++v) k.sets[(size_t)i].push_back(kw_code_to_leaf(*k.dict[i], l, f.values[v]));
      f.values = k.sets[(size_t)i].data();
    }
    x.agg_filters = k.filters.data();
  }
  return x;
}

static int32_t ix_n_distinct(const nrtgpu_index* ix, int32_t c) {
  return (size_t)c < ix->col_n_distinct.size() ? ix->col_n_distinct[(size_t)c] : 0;
}

// the reader-wide dictionary of `column` (built on `st` the first time it is asked for)
static int searcher_dict(nrtgpu_searcher* s, int32_t column, cudaStream_t st, const ReaderDict** out) {
  auto it = s->dicts.find(column);
  if (it != s->dicts.end()) { *out = it->second.get(); return NRTGPU_OK; }
  std::unique_ptr<ReaderDict> d(new ReaderDict);
  size_t total = 0;
  for (const nrtgpu_index* ix : s->leaves) total += (size_t)ix_n_distinct(ix, column);
  int rc;
  if ((rc = d->values.alloc(std::max<size_t>(total, 1)))) return rc;
  size_t at = 0;
  for (const nrtgpu_index* ix : s->leaves) {   // the leaves' dictionaries one after the other, then sorted and deduplicated
    const size_t nd = (size_t)ix_n_distinct(ix, column);
    if (nd) NRT_CUDA_TRY(cudaMemcpyAsync(d->values.p + at, ix_col_distinct(ix, column), nd * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
    at += nd;
  }
  if (total) {
    thrust::sort(thrust::cuda::par.on(st), d->values.p, d->values.p + total);
    d->n = (int32_t)(thrust::unique(thrust::cuda::par.on(st), d->values.p, d->values.p + total) - d->values.p);
  }
  d->values.n = (size_t)d->n;
  DevBuf<uint32_t> map;
  for (const nrtgpu_index* ix : s->leaves) {
    const int32_t nd = ix_n_distinct(ix, column);
    d->own.emplace_back(new DevBuf<uint32_t>);
    if (nd == d->n || nd == 0) { d->codes.push_back(ix_col_code(ix, column)); continue; }   // codes already reader-wide, or all 0
    DevBuf<uint32_t>& own = *d->own.back();
    if ((rc = map.alloc((size_t)nd)) || (rc = own.alloc((size_t)ix->n_docs))) return rc;
    dict_map_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, st>>>(ix_col_distinct(ix, column), nd, d->values.p, d->n, map.p);
    NRT_CUDA_TRY(cudaGetLastError());
    dict_remap_kernel<<<(unsigned)((ix->n_docs + 255) / 256), 256, 0, st>>>(ix_col_code(ix, column), ix->n_docs, map.p, own.p);
    NRT_CUDA_TRY(cudaGetLastError());
    NRT_CUDA_TRY(cudaStreamSynchronize(st));   // the map is reused by the next leaf
    d->codes.push_back(own.p);
  }
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  *out = d.get();
  s->dicts[column] = std::move(d);
  return NRTGPU_OK;
}

// the flags word of a record: relation GTE, terminated early, hit timeout
static void unpack_record_flags(const int32_t* flags, int32_t nq, uint8_t* out_relation, uint8_t* out_hit_timeout,
                                uint8_t* out_terminated_early) {
  for (int q = 0; q < nq; ++q) {
    if (out_relation) out_relation[q] = (uint8_t)(flags[q] & 1);
    if (out_terminated_early) out_terminated_early[q] = (uint8_t)((flags[q] >> 1) & 1);
    if (out_hit_timeout) out_hit_timeout[q] = (uint8_t)((flags[q] >> 2) & 1);
  }
}

static int searcher_merge_scored(nrtgpu_searcher* s, int32_t nq, int32_t top_k, void* stream, int32_t* out_docs, float* out_scores,
                                 int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                                 uint8_t* out_terminated_early);

// Score-ranked search over the leaves: run(l, d_record) leaves leaf l's page in its packed score record
// (nrtgpu_packed_words), the records are merged on the device (TopDocs.merge: nrtgpu_merge_topk_packed) and the merged
// page is copied to the host outputs (any may be NULL). The first failing leaf's code is returned and no output is written.
template <class Fn>
static int searcher_scored(nrtgpu_searcher* s, const char* fn, int32_t nq, int32_t top_k, void* stream, Fn&& run, int32_t* out_docs,
                           float* out_scores, int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation,
                           uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": NULL searcher");
  if (nq <= 0 || top_k <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, std::string(fn) + ": nq and top_k must be > 0");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  std::lock_guard<std::mutex> g(s->mu);
  const int64_t words = nrtgpu_packed_words(nq, top_k);
  const int n_leaves = (int)s->leaves.size();
  int rc;
  if ((rc = s->records.alloc((size_t)words * n_leaves)) || (rc = s->merged.alloc((size_t)words))) return rc;
  for (int l = 0; l < n_leaves; ++l)
    if ((rc = run(l, s->records.p + (size_t)l * words))) return rc;
  return searcher_merge_scored(s, nq, top_k, stream, out_docs, out_scores, out_counts, out_total_hits, out_relation, out_hit_timeout,
                               out_terminated_early);
}

// the tail of searcher_scored: the leaves' records in s->records merged on the device, the merged page to the host outputs
static int searcher_merge_scored(nrtgpu_searcher* s, int32_t nq, int32_t top_k, void* stream, int32_t* out_docs, float* out_scores,
                                 int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                                 uint8_t* out_terminated_early) {
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t words = nrtgpu_packed_words(nq, top_k);
  const int n_leaves = (int)s->leaves.size();
  int rc;
  if ((rc = nrtgpu_merge_topk_packed(s->ctx, n_leaves, nq, top_k, s->records.p, s->merged.p, stream))) return rc;
  s->host.resize((size_t)words);
  NRT_CUDA_TRY(cudaMemcpyAsync(s->host.data(), s->merged.p, (size_t)words * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  const int64_t n = (int64_t)nq * top_k;
  int64_t w = 2 * n + 2ll * nq; w = (w + 1) & ~1ll;
  if (out_docs) std::memcpy(out_docs, s->host.data(), (size_t)n * 4);
  if (out_scores) std::memcpy(out_scores, s->host.data() + n, (size_t)n * 4);
  if (out_counts) std::memcpy(out_counts, s->host.data() + 2 * n, (size_t)nq * 4);
  unpack_record_flags(s->host.data() + 2 * n + nq, nq, out_relation, out_hit_timeout, out_terminated_early);
  if (out_total_hits) std::memcpy(out_total_hits, s->host.data() + w, (size_t)nq * 8);
  return NRTGPU_OK;
}

// a kNN page of one leaf (host pages of the single-image search) uploaded into a packed score record; a leaf without
// vectors contributes an empty page
template <class Fn>
static int knn_leaf_record(nrtgpu_index* ix, int32_t nq, int32_t k, void* stream, int32_t* d_record, Fn&& search) {
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = (size_t)nq * k;
  NRT_CUDA_TRY(cudaMemsetAsync(d_record, 0, (size_t)nrtgpu_packed_words(nq, k) * sizeof(int32_t), st));
  if (ix->vec_dims <= 0) return NRTGPU_OK;
  std::vector<int32_t> docs(n), counts((size_t)nq);
  std::vector<float> scores(n);
  if (int rc = search(docs.data(), scores.data(), counts.data())) return rc;
  NRT_CUDA_TRY(cudaMemcpyAsync(d_record, docs.data(), n * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_record + n, scores.data(), n * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(d_record + 2 * n, counts.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));   // the staging vectors are freed on return
  return NRTGPU_OK;
}

static int searcher_aggs(nrtgpu_searcher* s, const char* fn, const BatchRequest& r, const nrtgpu_aggregation_result* results,
                         const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs, float* out_scores,
                         int32_t* out_counts, int64_t* out_total_hits);

static bool searcher_has_vectors(const nrtgpu_searcher* s) {
  for (const nrtgpu_index* ix : s->leaves) if (ix->vec_dims > 0) return true;
  return false;
}

// two sort orders rank by the same Sort: every field's kind and direction, and a column or keyword field's column,
// selector and missing value
static bool same_sort(const nrtgpu_sort_order* a, const nrtgpu_sort_order* b) {
  if (a->n_fields != b->n_fields) return false;
  for (int i = 0; i < a->n_fields; ++i) {
    const nrtgpu_sort_field &x = a->spec[i], &y = b->spec[i];
    if (x.kind != y.kind || (x.reverse != 0) != (y.reverse != 0)) return false;
    if ((x.kind == NRTGPU_SORT_COLUMN || x.kind == NRTGPU_SORT_KEYWORD) &&
        (x.column != y.column || x.selector != y.selector || x.missing_value != y.missing_value)) return false;
  }
  return true;
}

extern "C" {

int nrtgpu_searcher_create(nrtgpu_ctx* ctx, nrtgpu_index* const* leaves, int32_t n_leaves, nrtgpu_searcher** out) {
  if (!ctx || !leaves || n_leaves <= 0 || !out) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_create: bad argument");
  std::unique_ptr<nrtgpu_searcher> s(new nrtgpu_searcher);
  s->ctx = ctx;
  for (int i = 0; i < n_leaves; ++i) {
    if (!leaves[i] || leaves[i]->ctx != ctx) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_create: leaf of another context");
    s->leaves.push_back(leaves[i]);
  }
  *out = s.release();
  return NRTGPU_OK;
}

int nrtgpu_searcher_close(nrtgpu_searcher* s) { delete s; return NRTGPU_OK; }

int nrtgpu_searcher_keyword_seek(nrtgpu_searcher* s, int32_t column, const uint8_t* bytes, int32_t len, int64_t* code) {
  if (!s || !code || (!bytes && len > 0) || len < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_seek: bad argument");
  if (!searcher_has_kw(s, column)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_seek: keyword column out of range");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  std::lock_guard<std::mutex> g(s->mu);
  const ReaderDict* d = nullptr;
  if (int rc = searcher_kw_dict(s, column, nullptr, &d)) return rc;
  *code = keyword_seek_code(d->bytes.data(), d->off.data(), d->n, bytes, len);
  return NRTGPU_OK;
}

int nrtgpu_searcher_keyword_range(nrtgpu_searcher* s, int32_t column, const uint8_t* lower, int32_t lower_len, const uint8_t* upper,
                                  int32_t upper_len, int32_t flags, int64_t* lo, int64_t* hi) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_range: NULL searcher");
  if (!searcher_has_kw(s, column)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_range: keyword column out of range");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  std::lock_guard<std::mutex> g(s->mu);
  const ReaderDict* d = nullptr;
  if (int rc = searcher_kw_dict(s, column, nullptr, &d)) return rc;
  return keyword_range_codes(d->bytes.data(), d->off.data(), d->n, lower, lower_len, upper, upper_len, flags, lo, hi);
}

int nrtgpu_searcher_keyword_term(nrtgpu_searcher* s, int32_t column, int32_t ord, uint8_t* out, int32_t cap, int32_t* len,
                                 int32_t* n_terms) {
  if (!s || !len) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_term: NULL argument");
  if (!searcher_has_kw(s, column)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_term: keyword column out of range");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  std::lock_guard<std::mutex> g(s->mu);
  const ReaderDict* d = nullptr;
  if (int rc = searcher_kw_dict(s, column, nullptr, &d)) return rc;
  if (n_terms) *n_terms = d->n;
  *len = 0;
  if (ord == -1 && n_terms) return NRTGPU_OK;
  if (ord < 0 || ord >= d->n) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_keyword_term: ordinal out of range");
  copy_term(d->bytes, d->off, ord, out, cap, len);
  return NRTGPU_OK;
}

int nrtgpu_searcher_search_bool(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold,
                                int32_t flags, const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs,
                                float* out_scores, int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation) {
  if (!s || !out_docs || !out_scores || !out_counts) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_bool: NULL argument");
  if (nq <= 0 || top_k <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_bool: nq and top_k must be > 0");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> g(s->mu);
  const int64_t words = nrtgpu_packed_words(nq, top_k);
  const int n_leaves = (int)s->leaves.size();
  int rc;
  if ((rc = s->records.alloc((size_t)words * n_leaves)) || (rc = s->merged.alloc((size_t)words))) return rc;
  std::vector<const ReaderDict*> kw;   // keyword clauses: each leaf receives their codes in its own dictionary
  std::vector<nrtgpu_clause> leaf_clauses;
  bool any_kw = false;
  if ((rc = searcher_kw_clauses(s, clauses, n_clauses, st, &kw, &any_kw))) return rc;
  for (int l = 0; l < n_leaves; ++l) {   // every leaf runs the whole batch (LeafCollector per segment), results stay on the device
    const nrtgpu_clause* cl = any_kw ? kw_leaf_clauses(kw, clauses, n_clauses, (size_t)l, leaf_clauses) : clauses;
    if ((rc = nrtgpu_search_bool_packed(s->leaves[(size_t)l], cl, n_clauses, queries, nq, top_k, total_hits_threshold, flags, limits,
                                        stream, s->records.p + (size_t)l * words))) return rc;
  }
  // TopDocs.merge over the leaves (LazyQueueTopScoreDocCollectorManager.java:137-144)
  if ((rc = nrtgpu_merge_topk_packed(s->ctx, n_leaves, nq, top_k, s->records.p, s->merged.p, stream))) return rc;
  s->host.resize((size_t)words);
  NRT_CUDA_TRY(cudaMemcpyAsync(s->host.data(), s->merged.p, (size_t)words * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  const int64_t n = (int64_t)nq * top_k;
  int64_t w = 2 * n + 2ll * nq; w = (w + 1) & ~1ll;
  std::memcpy(out_docs, s->host.data(), (size_t)n * 4);
  std::memcpy(out_scores, s->host.data() + n, (size_t)n * 4);
  std::memcpy(out_counts, s->host.data() + 2 * n, (size_t)nq * 4);
  if (out_relation) for (int q = 0; q < nq; ++q) out_relation[q] = (uint8_t)(s->host[(size_t)(2 * n + nq + q)] & 1);
  if (out_total_hits) std::memcpy(out_total_hits, s->host.data() + w, (size_t)nq * 8);
  return NRTGPU_OK;
}

int nrtgpu_searcher_search_sorted_fields(nrtgpu_searcher* s, const nrtgpu_sort_order* const* orders, int32_t n_orders,
                                         const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_query* queries, int32_t nq,
                                         int32_t top_k, int32_t flags, const int64_t* after_values,
                                         const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs,
                                         int64_t* out_sort_values, int32_t* out_counts, int64_t* out_total_hits,
                                         uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  if (!s || !orders) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: NULL argument");
  const int n_leaves = (int)s->leaves.size();
  if (n_orders != n_leaves) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: one sort order per leaf is needed");
  for (int l = 0; l < n_leaves; ++l) {
    if (!orders[l]) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: NULL sort order");
    if (orders[l]->ix != s->leaves[(size_t)l])
      NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: the sort order of leaf " + std::to_string(l) + " was made on another index");
    if (!same_sort(orders[l], orders[0])) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: the leaves' sort orders are of different Sorts");
  }
  if (nq <= 0 || top_k <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_sorted_fields: nq and top_k must be > 0");
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> g(s->mu);
  const int32_t nf = orders[0]->n_fields;
  const SortedRecordLayout L = sorted_record_layout(nq, top_k, nf);
  int rc;
  // keyword fields: reader-wide after codes are checked against the union, then given to each leaf in its own dictionary,
  // and each leaf's hit values are mapped to the union before the merge
  const ReaderDict* kw[kMaxSortFields] = {};
  std::vector<std::array<const uint32_t*, kMaxSortFields>> kw_maps;
  if ((rc = searcher_sort_kw(s, orders[0], st, kw, &kw_maps))) return rc;
  bool any_kw = false;
  int32_t kw_n[kMaxSortFields] = {};
  for (int j = 0; j < nf; ++j) if (kw[j]) { any_kw = true; kw_n[j] = kw[j]->n; }
  if (any_kw && after_values && queries &&
      (rc = check_keyword_after(orders[0], after_values, queries, nq, "nrtgpu_searcher_search_sorted_fields", kw_n))) return rc;
  if ((rc = s->records.alloc((size_t)L.words * n_leaves)) || (rc = s->merged.alloc((size_t)L.words))) return rc;
  std::vector<const ReaderDict*> kw_cl;   // keyword clauses, mapped per leaf as the after codes are
  std::vector<nrtgpu_clause> leaf_clauses;
  bool any_kw_cl = false;
  if ((rc = searcher_kw_clauses(s, clauses, n_clauses, st, &kw_cl, &any_kw_cl))) return rc;
  std::vector<int64_t> leaf_after;
  for (int l = 0; l < n_leaves; ++l) {   // every leaf pages after the same reader-wide FieldDoc
    const int64_t* av = after_values;
    if (any_kw && after_values) {
      leaf_after.assign(after_values, after_values + (size_t)nq * nf);
      for (int j = 0; j < nf; ++j)
        if (kw[j])
          for (int q = 0; q < nq; ++q) leaf_after[(size_t)q * nf + j] = kw_code_to_leaf(*kw[j], (size_t)l, after_values[(size_t)q * nf + j]);
      av = leaf_after.data();
    }
    int32_t* rec = s->records.p + (size_t)l * L.words;
    const nrtgpu_clause* cl = any_kw_cl ? kw_leaf_clauses(kw_cl, clauses, n_clauses, (size_t)l, leaf_clauses) : clauses;
    if ((rc = nrtgpu_search_sorted_fields_packed(s->leaves[(size_t)l], orders[l], cl, n_clauses, queries, nq, top_k, flags, av,
                                                 limits, stream, rec))) return rc;
    if (any_kw && (rc = sort_kw_values_to_union(kw_maps[(size_t)l].data(), nf, reinterpret_cast<int64_t*>(rec + L.values),
                                                (int64_t)nq * top_k, st))) return rc;
  }
  // TopFieldDocs.merge over the leaves
  if ((rc = nrtgpu_merge_sorted_packed(s->ctx, orders[0]->spec, nf, n_leaves, nq, top_k, s->records.p, s->merged.p, stream))) return rc;
  s->host.resize((size_t)L.words);
  NRT_CUDA_TRY(cudaMemcpyAsync(s->host.data(), s->merged.p, (size_t)L.words * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  const int64_t n = (int64_t)nq * top_k;
  if (out_docs) std::memcpy(out_docs, s->host.data(), (size_t)n * 4);
  if (out_sort_values) std::memcpy(out_sort_values, s->host.data() + L.values, (size_t)n * nf * 8);
  if (out_counts) std::memcpy(out_counts, s->host.data() + L.counts, (size_t)nq * 4);
  unpack_record_flags(s->host.data() + L.flags, nq, out_relation, out_hit_timeout, out_terminated_early);
  if (out_total_hits) std::memcpy(out_total_hits, s->host.data() + L.totals, (size_t)nq * 8);
  return NRTGPU_OK;
}

int nrtgpu_searcher_search_tree_phrases(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                                        int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                        const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                                        int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                                        const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores,
                                        int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation,
                                        uint8_t* out_hit_timeout, uint8_t* out_terminated_early) {
  if (n_nodes < 0 || (n_nodes > 0 && !nodes)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_search_tree: bad nodes");
  BatchRequest r = tree_request(clauses, n_clauses, nodes, n_nodes, queries, nq, top_k, total_hits_threshold, flags);
  int rc = phrase_request(&r, phrases, n_phrases, phrase_terms, n_phrase_terms);
  if (rc) return rc;
  r.unions = true;
  KwLeafRequest kw;
  return searcher_scored(s, "nrtgpu_searcher_search_tree_phrases", nq, top_k, stream, [&](int l, int32_t* d_record) {
    // (the leaves run in order under the searcher's lock: the first prepares the keyword codes of every leaf)
    if (l == 0) { if (int rc2 = searcher_kw_request(s, r, (cudaStream_t)stream, &kw)) return rc2; }
    SearchOut o; o.d_record = d_record; o.record_limits = true;
    return search_bool_impl(s->leaves[(size_t)l], kw_leaf_request(kw, r, (size_t)l), limits, stream, o);
  }, out_docs, out_scores, out_counts, out_total_hits, out_relation, out_hit_timeout, out_terminated_early);
}

int nrtgpu_searcher_search_knn(nrtgpu_searcher* s, const float* queries, int32_t nq, int32_t k, const float* boosts,
                               const uint8_t* filter, void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts) {
  if (!s || !queries || !out_docs || !out_scores || !out_counts) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn: NULL argument");
  if (!searcher_has_vectors(s)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn: no leaf has a vector field");
  if (nq <= 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn: nq must be > 0");
  if (k <= 0 || k > kMaxTopK) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn: k out of range");
  if (!knn_boosts_valid(boosts, nq)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn: a boost must be finite and >= 0");
  return searcher_scored(s, "nrtgpu_searcher_search_knn", nq, k, stream, [&](int l, int32_t* d_record) {
    nrtgpu_index* ix = s->leaves[(size_t)l];
    return knn_leaf_record(ix, nq, k, stream, d_record, [&](int32_t* d, float* sc, int32_t* c) {
      return nrtgpu_search_knn(ix, queries, nq, k, boosts, filter ? filter + ix->doc_base : nullptr, stream, d, sc, c);
    });
  }, out_docs, out_scores, out_counts, nullptr, nullptr, nullptr, nullptr);
}

int nrtgpu_searcher_search_knn_filtered(nrtgpu_searcher* s, const float* queries, int32_t nq, int32_t k, const float* boosts,
                                        const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filters,
                                        int32_t n_filters, const int32_t* filter_of, void* stream, int32_t* out_docs,
                                        float* out_scores, int32_t* out_counts) {
  if (!s || !queries || !out_docs || !out_scores || !out_counts || !filter_of || (n_filters > 0 && !filters))
    NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn_filtered: NULL argument");
  if (!searcher_has_vectors(s)) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn_filtered: no leaf has a vector field");
  if (nq <= 0 || n_filters < 0) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn_filtered: nq must be > 0 and n_filters >= 0");
  if (k <= 0 || k > kMaxTopK) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_knn_filtered: k out of range");
  std::vector<const ReaderDict*> kw;
  std::vector<nrtgpu_clause> leaf_clauses;
  bool any_kw = false;
  return searcher_scored(s, "nrtgpu_searcher_search_knn_filtered", nq, k, stream, [&](int l, int32_t* d_record) {
    // (the leaves run in order under the searcher's lock: the first checks the keyword clauses against the union)
    if (l == 0) { if (int rc = searcher_kw_clauses(s, filter_clauses, n_filter_clauses, (cudaStream_t)stream, &kw, &any_kw)) return rc; }
    nrtgpu_index* ix = s->leaves[(size_t)l];
    const nrtgpu_clause* cl = any_kw ? kw_leaf_clauses(kw, filter_clauses, n_filter_clauses, (size_t)l, leaf_clauses) : filter_clauses;
    return knn_leaf_record(ix, nq, k, stream, d_record, [&](int32_t* d, float* sc, int32_t* c) {
      return nrtgpu_search_knn_filtered(ix, queries, nq, k, boosts, cl, n_filter_clauses, filters, n_filters, filter_of,
                                        stream, d, sc, c);
    });
  }, out_docs, out_scores, out_counts, nullptr, nullptr, nullptr, nullptr);
}

int nrtgpu_searcher_search_bool_aggs_nested(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                            const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                            const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                            const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs,
                                            float* out_scores, int32_t* out_counts, int64_t* out_total_hits) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_bool_aggs_nested: NULL searcher");
  return nrtgpu_searcher_search_bool_aggs_filtered(s, clauses, n_clauses, queries, nq, top_k, flags, aggs, n_aggs, results, nested,
                                                   n_nested, nested_results, nullptr, nullptr, 0, nullptr, 0, stream, out_docs,
                                                   out_scores, out_counts, out_total_hits);
}

int nrtgpu_searcher_search_bool_aggs_filtered(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                              const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                              const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                              const nrtgpu_aggregation_result* results, const nrtgpu_nested_aggregation* nested,
                                              int32_t n_nested, const nrtgpu_nested_result* nested_results,
                                              const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                              int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                                              int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores,
                                              int32_t* out_counts, int64_t* out_total_hits) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_bool_aggs_filtered: NULL searcher");
  return nrtgpu_searcher_search_bool_aggs_sorted_hits(s, clauses, n_clauses, queries, nq, top_k, flags, aggs, n_aggs, results, nested,
                                                      n_nested, nested_results, nullptr, agg_filters, filter_clauses, n_filter_clauses,
                                                      filter_queries, n_filter_queries, stream, out_docs, out_scores, out_counts,
                                                      out_total_hits);
}

// Aggregations over the leaves (searcher_aggs)
int nrtgpu_searcher_search_bool_aggs_sorted_hits(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                                 const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                                 const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                                 const nrtgpu_aggregation_result* results,
                                                 const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                                 const nrtgpu_nested_result* nested_results, const nrtgpu_nested_sort* nested_sorts,
                                                 const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                                 int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                                                 int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores,
                                                 int32_t* out_counts, int64_t* out_total_hits) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_bool_aggs_sorted_hits: NULL searcher");
  BatchRequest r{clauses, n_clauses, queries, nq, top_k, INT32_MAX, flags};
  int rc = aggs_request(&r, aggs, n_aggs, results, nested, n_nested, nested_results, nested_sorts, agg_filters, filter_clauses,
                        n_filter_clauses, filter_queries, n_filter_queries);
  if (rc) return rc;
  return searcher_aggs(s, "nrtgpu_searcher_search_bool_aggs_sorted_hits", r, results, nested_results, stream, out_docs, out_scores,
                       out_counts, out_total_hits);
}

int nrtgpu_searcher_search_tree_aggs(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                                     int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                     const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                                     int32_t nq, int32_t top_k, int32_t flags, const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                     const nrtgpu_aggregation_result* results, const nrtgpu_nested_aggregation* nested,
                                     int32_t n_nested, const nrtgpu_nested_result* nested_results,
                                     const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                                     const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                                     const nrtgpu_query* filter_queries, int32_t n_filter_queries, void* stream, int32_t* out_docs,
                                     float* out_scores, int32_t* out_counts, int64_t* out_total_hits) {
  if (!s) NRT_FAIL(NRTGPU_ERR_INVALID, "nrtgpu_searcher_search_tree_aggs: NULL searcher");
  BatchRequest r;
  int rc = tree_aggs_request(&r, clauses, n_clauses, nodes, n_nodes, phrases, n_phrases, phrase_terms, n_phrase_terms, queries, nq, top_k,
                             flags, aggs, n_aggs, results, nested, n_nested, nested_results, nested_sorts, agg_filters, filter_clauses,
                             n_filter_clauses, filter_queries, n_filter_queries);
  if (rc) return rc;
  return searcher_aggs(s, "nrtgpu_searcher_search_tree_aggs", r, results, nested_results, stream, out_docs, out_scores, out_counts,
                       out_total_hits);
}

#include "batcher.inc"

}  // extern "C"

// The collector searches over the leaves (request r from aggs_request; fn names the entry point in refusals): every leaf's
// batch counts into one set of reader-wide tables through its codes renumbered to the column's reader-wide dictionary
// (searcher_dict) and tests its own image's filter rows; the selection and the nested top hits then run once on them
// (sorted top hits: per leaf, then merged; batch_nested_top_hits)
static int searcher_aggs(nrtgpu_searcher* s, const char* fn, const BatchRequest& r, const nrtgpu_aggregation_result* results,
                         const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs, float* out_scores,
                         int32_t* out_counts, int64_t* out_total_hits) {
  const nrtgpu_aggregation* aggs = r.aggs;
  const nrtgpu_nested_aggregation* nested = r.nested;
  const int32_t nq = r.nq, top_k = r.top_k, n_aggs = r.n_aggs, n_nested = r.n_nested;
  int rc;
  if ((rc = check_nested_sorts(fn, r, s->leaves.data(), (int)s->leaves.size()))) return rc;
  NRT_CUDA_TRY(cudaSetDevice(s->ctx->device));
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> g(s->mu);
  const int n_leaves = (int)s->leaves.size();
  KwLeafRequest kw;   // keyword clauses and sets: reader-wide codes, checked against the union, mapped per leaf
  if ((rc = searcher_kw_request(s, r, st, &kw))) return rc;
  std::vector<KwLeafRequest> kw_leaf((size_t)n_leaves, kw);   // (each leaf's request points into its own copies)
  std::vector<BatchRequest> lr;
  for (int l = 0; l < n_leaves; ++l) lr.push_back(kw_leaf_request(kw_leaf[(size_t)l], r, (size_t)l));
  {   // every refusal of the single-image call, on every leaf's columns, before any batch is built
    CompiledBatch cb;
    for (int l = 0; l < n_leaves; ++l)
      if ((rc = compile_batch(s->leaves[(size_t)l]->dict(), lr[(size_t)l], &cb))) return rc;
  }
  // the reader-wide dictionaries, and the table limits of the single-image call at their size
  const ReaderDict* dict[kMaxAggs] = {};
  int32_t n_buckets[kMaxAggs] = {};
  for (int i = 0; i < n_aggs; ++i) {
    n_buckets[i] = 1;   // (a filter's one bucket)
    if (aggs[i].kind != NRTGPU_AGG_TERMS) continue;
    if ((rc = agg_keyword(aggs[i]) ? searcher_kw_dict(s, aggs[i].column, st, &dict[i]) : searcher_dict(s, aggs[i].column, st, &dict[i])))
      return rc;
    n_buckets[i] = dict[i]->n;
    if ((int64_t)nq * n_buckets[i] * 4 > (2ll << 30))
      NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "terms aggregation: batch x distinct values exceeds the 2 GB count table");
  }
  for (int j = 0; j < n_nested; ++j)
    if (nested[j].kind != NRTGPU_AGG_TOP_HITS && (int64_t)nq * n_buckets[nested[j].parent] * 8 > (2ll << 30))
      NRT_FAIL(NRTGPU_ERR_UNSUPPORTED, "nested aggregation: batch x distinct values exceeds the 2 GB table");
  // one pooled workspace per leaf, held until the nested top hits of every leaf are collected
  std::vector<std::unique_ptr<WorkspaceLease>> ws;
  std::vector<nrtgpu_batch*> bs;
  for (nrtgpu_index* ix : s->leaves) { ws.emplace_back(new WorkspaceLease(ix)); bs.push_back(ws.back()->b); }
  const int64_t words = nrtgpu_packed_words(nq, top_k);
  if ((rc = s->records.alloc((size_t)words * n_leaves)) || (rc = s->merged.alloc((size_t)words))) return rc;
  for (int l = 0; l < n_leaves; ++l) {
    if ((rc = batch_build(bs[(size_t)l], s->leaves[(size_t)l], lr[(size_t)l], st)) || (rc = batch_set_limits(bs[(size_t)l], nullptr, st)) ||
        (rc = nrtgpu_batch_bind_packed(bs[(size_t)l], s->records.p + (size_t)l * words))) return rc;
  }
  // sorted top hits by a Sort with keyword fields: each leaf's hit values are mapped to the reader-wide dictionaries
  for (int j = 0; j < n_nested && r.nested_sorts && n_leaves > 1; ++j) {
    const nrtgpu_sort_order* const* orders = r.nested_sorts[j].orders;
    if (!orders || nested[j].kind != NRTGPU_AGG_TOP_HITS) continue;
    const ReaderDict* kw[kMaxSortFields] = {};
    std::vector<std::array<const uint32_t*, kMaxSortFields>> maps;
    if ((rc = searcher_sort_kw(s, orders[0], st, kw, &maps))) return rc;
    for (int l = 0; l < n_leaves; ++l) {
      std::vector<std::array<const uint32_t*, kMaxSortFields>>& m = bs[(size_t)l]->nest_kw_map;
      m.resize((size_t)n_nested, std::array<const uint32_t*, kMaxSortFields>{});
      m[(size_t)j] = maps[(size_t)l];
    }
  }
  // the reader-wide tables live in leaf 0's workspace and are reset once; every leaf counts into them with its own codes
  AggTables t = {};
  if ((rc = batch_agg_tables(bs[0], n_buckets, st, &t))) return rc;
  for (int l = 0; l < n_leaves; ++l) {
    AggTables& x = bs[(size_t)l]->agg_tab;
    x = t;
    for (int i = 0; i < n_aggs; ++i)
      if (dict[i]) {
        x.codes[i] = dict[i]->codes[(size_t)l]; x.distinct[i] = dict[i]->values.p;
        if (agg_keyword(aggs[i])) {   // reader-wide ordinals, per doc (SORTED) or per value behind the leaf's doc offsets
          x.distinct[i] = nullptr;
          x.offsets[i] = s->leaves[(size_t)l]->kw[(size_t)aggs[i].column]->doc_off.p;
        }
      }
    bs[(size_t)l]->agg_shared = true;
  }
  for (int l = 0; l < n_leaves; ++l)
    if ((rc = nrtgpu_batch_run(bs[(size_t)l], stream))) return rc;
  if ((rc = batch_fetch_aggs(bs.data(), n_leaves, st, results, n_nested > 0 ? nested_results : nullptr))) return rc;
  // TopDocs.merge of the leaves' pages; totalHits is exact (every match is counted) and summed over the leaves
  return searcher_merge_scored(s, nq, top_k, stream, out_docs, out_scores, out_counts, out_total_hits, nullptr, nullptr, nullptr);
}
