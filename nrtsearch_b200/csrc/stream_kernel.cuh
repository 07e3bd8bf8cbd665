// posting_stream_kernel -- the batched BooleanQuery engine for queries of <= 4 term clauses (DESIGN.md 4.1).
//
// One work item = (query, 524,288-doc slice). Everything a work item reads arrives by TMA or is index-time data:
//   * posting lists are STREAMED through per-clause rings in shared memory filled by 1-D TMA bulk copies
//     (cp.async.bulk.shared.global + mbarrier complete_tx, SASS UBLKCP) issued by the lanes of warp 0;
//   * run boundaries come from granule bounds (postings of every list below each 1024-doc granule: index-time skip
//     data for long lists, one lower_bound per granule for short ones), so the sweep never searches to find them;
//   * exact BM25 floats tbl[slot][tf][norm] and the tf-pattern bound ubt[] are computed once per batch and query
//     (query_tables_kernel) and pulled in with one TMA copy: no IEEE division per posting;
//   * for pure disjunctions ubt[] rejects, with one shared-memory load, every doc whose best possible score is below
//     the running threshold theta (rank-safe: the bound is the same float expression at the shortest field length
//     present in the index); survivors are appended unscored and scored together at the buffer flush;
//   * no barrier inside a pass: a thread whose candidate does not fit the buffer parks it, the CTA flushes once, and
//     parked threads resume.
// Three sweep modes per work item: window (scatter tf bytes into an 8K-doc word array -> owners emit), tf-plane (a
// dense non-essential list is a TMA copy of its direct-address bytes instead of a scatter) and sparse (short lists
// merged by granule-narrowed binary search of each other's ring segments, plane bytes gathered from L2).
// Results are bit-identical to the exhaustive oracle; totalHits are exact until MAXSCORE prunes (then a lower bound
// with relation GREATER_THAN_OR_EQUAL_TO, as in the reference).
#pragma once
#include <cstddef>
#include "bool_kernel.cuh"

namespace nrtgpu {
namespace v2 {

constexpr int kT = 4;
#ifndef NRT_STREAM_CTAS
#define NRT_STREAM_CTAS 2   // two independent CTAs per SM: one CTA's barrier waits are filled by the other's warps
#endif
constexpr int kCtasPerSm = NRT_STREAM_CTAS;
constexpr int kLogCH = 9;
constexpr int kCH = 1 << kLogCH;      // postings per chunk
constexpr int kMaxNCH = 32;           // largest ring (chunks, power of two)
#if NRT_STREAM_CTAS == 1
constexpr int kW = 16384;             // docs per window (one 32-bit word each)
constexpr int kPool = 40;             // chunks in the CTA's ring pool, shared by the term clauses
constexpr int kMinNCH = 8;            // a ring always holds one full granule (<= 2048 postings) plus alignment slack
constexpr int kLogGran = 11;          // posting bounds are precomputed per (query, clause) at 2048-doc granules
constexpr int kSliceDocs = 1 << 20;   // docs per work item
constexpr int kCand = 2048;
constexpr int kTfTab = 4;             // table rows tf = 0..kTfTab (row 0 = 0.0f)
#else                                 // two CTAs per SM: half the window / ring pool / candidate buffer each
constexpr int kW = 8192;
constexpr int kPool = 18;
constexpr int kMinNCH = 4;            // one 1024-doc granule (<= 1024 postings = 2 chunks) plus alignment slack
constexpr int kLogGran = 10;
constexpr int kSliceDocs = 1 << 19;
constexpr int kCand = 1024;
constexpr int kTfTab = 2;
#endif
constexpr int kMaxTopKStream = kCand / 2;   // larger top_k goes through bool_window_kernel
#ifndef NRT_STREAM_THREADS
#define NRT_STREAM_THREADS (NRT_STREAM_CTAS == 1 ? 512 : 256)   // 64K registers per SM / 128 per thread
#endif
constexpr int kThreads = NRT_STREAM_THREADS;   // one CTA per SM
constexpr int kGran = 1 << kLogGran;
static_assert((kThreads & (kThreads - 1)) == 0, "the round-robin posting deal masks with kThreads - 1");
constexpr int kWinGran = kW / kGran;  // a window spans up to 8 granules
constexpr int kUbt = 6 * 6 * 6 * 6;   // upper-bound table over min(tf, 5) of the four slots
constexpr uint32_t kChunkBytes = kCH * 4 + kCH;
constexpr int kQTabFloats = kT * (kTfTab + 1) * 256 + kUbt;   // per-query score + bound tables (query_tables_kernel)
#ifndef NRT_SPARSE_CAP
#define NRT_SPARSE_CAP 65536
#endif
constexpr int kSparseCap = NRT_SPARSE_CAP;   // (measured with granule-narrowed searches: 32K 5.84 ms, 64K 5.79, 128K 5.90)
#ifndef NRT_SPARSE_CAP_ALL
#define NRT_SPARSE_CAP_ALL 32768
#endif
constexpr int kSparseCapAll = NRT_SPARSE_CAP_ALL;          // ... when every list drives (no pruning): each posting pays the searches   // a list with at most this many postings in the slice can be merged by binary search
// sparse mode: doc chunks = pool_docs + the first kSparseExtra chunks' worth of the window array; their tf bytes = the rest
// of the window array + pool_f8
constexpr int kSparseExtra = (kW * 4) / (kCH * 4 + kCH) < 14 ? (kW * 4) / (kCH * 4 + kCH) : 14;
constexpr int kPoolSparse = kPool + kSparseExtra;
constexpr int kSparseF8Off = kSparseExtra * kCH * 4;   // byte offset of the sparse tf region inside the window array
static_assert(kW * 4 - kSparseF8Off + kPool * kCH >= kPoolSparse * kCH, "sparse tf chunks must fit behind the extra doc chunks");
constexpr int kWarmGran = 32;   // granules (32K docs) of the warm-up work item of a query
constexpr int kPlaneChunks = (2 * kW + kCH * 4 - 1) / (kCH * 4);   // pool chunks (doc part) lent to the two tf-plane buffers

struct StreamLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  const int32_t* work_query;
  const int32_t* work_slice;
  const uint32_t* gbounds;   // [nq][kT][n_gran+1]: postings of the clause with doc < g*kGran (relative to post_base)
  unsigned long long* mode_stats;  // optional (NRTGPU_DEBUG_MODES): [mode 0 window / 1 window+MAXSCORE / 2 sparse][cycles, items]
  const float* qtables;      // [nq][kQTabFloats]: tbl[slot][tf][norm] then ubt[tf pattern] of every query
  int32_t n_gran;
  int32_t n_work, n_slices, top_k;
  int32_t slice_docs;
  int64_t threshold;         // totalHitsThreshold (max(threshold, numHits)); INT32_MAX = exact counts, no list skipping
  int32_t* pruned;           // [nq] set to 1 when a work item skipped non-essential lists (relation GTE)
  uint64_t* theta;
  unsigned long long* total_hits;
  uint64_t* slice_keys;
  int32_t* slice_cnt;
};

struct alignas(128) StreamSmem {
  // ring pool (TMA destinations: 2 KB aligned doc chunks, 512 B tf chunks). Sparse mode has no window array and
  // extends the pool over it: doc chunks run on from pool_docs into slots, tf chunks start inside slots and run on
  // into pool_f8 -- the three arrays must stay in this order.
  int32_t pool_docs[kPool * kCH];
  uint32_t slots[kW];                    // window array: one 32-bit word (four tf bytes) per doc
  uint8_t pool_f8[kPool * kCH];
  uint64_t cand[kCand];                  // 16 KB
  float tbl[kT][kTfTab + 1][256];        // exact BM25 floats per (slot, tf, norm byte); row tf = 0 is +0.0f
  float ubt[kUbt];                       // score bound per tf pattern (directly after tbl: one TMA copy fills both)
  uint64_t full_bar[kPoolSparse];
  uint4 gb4[kSliceDocs / kGran + 1];      // 8 KB granule bounds of this slice, one 16-byte row {slot 0..3} per granule
  uint16_t nextg[kSliceDocs / kGran + 2]; // 1 KB window table: the window that starts at granule g ends at nextg[g]
  DevClause cl[kMaxClauses];
  DevQuery q;
  // per-slot stream descriptors (static after set-up; s_issued is owned by thread 0)
  const int32_t* s_gdocs[kT];
  const uint8_t* s_gf8[kT];
  int32_t s_r_begin[kT], s_r_end[kT], s_n_chunks[kT], s_issued[kT];
  int32_t s_field[kT], s_clause[kT];
  int32_t s_ring_base[kT], s_ring_nch[kT];   // first pool chunk and ring length (chunks, power of two) per slot
  uint32_t s_scoring[kT];
  const uint8_t* s_plane[kT];       // dense tf plane of the slot's term (NULL: none)
  int cand_count;
  unsigned long long hits0;         // the query's hit count when the work item started
  int n_keys;                       // entries [0, n_keys) of cand are keys kept by the last flush
  uint32_t ne_mask;                 // non-essential slots of this work item (MAXSCORE)
  int plane_slot;                   // non-essential slot served from its dense tf plane (-1: none)
  int sparse;                       // 1: sparse mode (no window array: lists merged by binary search, planes read from L2)
  uint32_t pserve_mask;             // sparse mode: non-essential slots read from their plane instead of being streamed
  uint64_t plane_bar[2];
  uint64_t tab_bar;
  unsigned long long theta;
};
static_assert(sizeof(StreamSmem) <= (kCtasPerSm == 1 ? 232448 : 115712), "StreamSmem exceeds the shared memory budget of sm_90");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ uint32_t presence4(uint32_t s) {
  return ((s & 0xffu) ? 1u : 0u) | ((s & 0xff00u) ? 2u : 0u) | ((s & 0xff0000u) ? 4u : 0u) | ((s & 0xff000000u) ? 8u : 0u);
}

__device__ __noinline__ float term_score_slow(const StreamLaunch& L, const DevClause& c, int32_t doc, uint32_t b, uint32_t nb) {
  float f = (b == 255u) ? exact_freq_slow<uint32_t>(L.ix, c, doc) : (float)b;
  return bm25_score(c.weight, f, __ldg(&L.ix.caches[c.field * 256 + nb]));
}

// Universal evaluation: any clause mix, any tf, deleted docs. Clause-order double sums, exactly as v1.
// Score combination follows Lucene's BooleanScorerSupplier: conjunction / disjunction sums are double,
// required+optional is ReqOptSumScorer's float add (msm == 0) or ConjunctionScorer's double add (msm > 0).
__device__ __noinline__ bool evaluate_doc_generic(const StreamLaunch& L, const StreamSmem& sm, int32_t doc, uint32_t slot,
                                                  float* out_score) {
  const DevQuery& q = sm.q;
  const uint32_t m = presence4(slot);
  if ((m & q.req_term_mask) != q.req_term_mask) return false;
  if (m & q.not_term_mask) return false;
  if (L.ix.live_bits && !((L.ix.live_bits[doc >> 5] >> (doc & 31)) & 1u)) return false;
  double must_sum = 0.0, should_sum = 0.0;
  int n_should = 0;
  int cur_field = -1;
  uint32_t nb = 1u;
  for (int i = 0; i < q.n_clauses; ++i) {
    const DevClause& c = sm.cl[i];
    bool present;
    float s = 0.0f;
    if (c.kind == NRTGPU_TERM) {
      const uint32_t b = (slot >> (8 * c.slot)) & 0xffu;
      present = b != 0;
      if (present && c.scoring) {
        if (c.field != cur_field) {
          cur_field = c.field;
          const uint8_t* nrm = L.ix.norms[c.field];
          nb = nrm ? (uint32_t)__ldg(nrm + doc) : 1u;
        }
        s = (b <= (uint32_t)kTfTab) ? sm.tbl[c.slot][b][nb] : term_score_slow(L, c, doc, b, nb);
      }
    } else if (c.kind == NRTGPU_RANGE_I64) {
      present = range_matches(L.ix, c.col, doc, c.lo, c.hi);
      s = c.weight;
    } else {
      present = true;
      s = c.weight;
    }
    if (!present) {
      if (c.occur == NRTGPU_MUST || c.occur == NRTGPU_FILTER) return false;
      continue;
    }
    switch (c.occur) {
      case NRTGPU_MUST: must_sum += (double)s; break;
      case NRTGPU_FILTER: break;
      case NRTGPU_SHOULD: should_sum += (double)s; ++n_should; break;
      default: return false;
    }
  }
  if (n_should < q.need_should) return false;
  float score;
  if (q.n_req == 0) score = (float)should_sum;
  else {
    float req = (float)must_sum;
    if (n_should == 0) score = req;
    else {
      float opt = (float)should_sum;
      score = (q.msm > 0) ? (float)((double)req + (double)opt) : __fadd_rn(req, opt);
    }
  }
  *out_score = score;
  return true;
}

// exact score of a doc of a PURE DISJUNCTION over one text field (every slot SHOULD): double sum in slot
// (= clause) order of the table floats; tf > kTfTab goes through the generic path
__device__ __noinline__ float score_disjunction_slow(const StreamLaunch& L, const StreamSmem& sm, int32_t doc, uint32_t v) {
  float s = 0.0f;
  evaluate_doc_generic(L, sm, doc, v, &s);
  return s;
}

__device__ __forceinline__ float score_disjunction(const StreamLaunch& L, const StreamSmem& sm, const uint8_t* norms0, int32_t doc,
                                                   uint32_t v) {
  const uint32_t b0 = v & 0xffu, b1 = (v >> 8) & 0xffu, b2 = (v >> 16) & 0xffu, b3 = v >> 24;
  if (max(max(b0, b1), max(b2, b3)) > (uint32_t)kTfTab) return score_disjunction_slow(L, sm, doc, v);
  const uint32_t nb = norms0 ? (uint32_t)__ldg(norms0 + doc) : 1u;
  double sum = (double)sm.tbl[0][b0][nb];   // rows tf = 0 hold +0.0f: adding them leaves the sum bit-identical
  sum += (double)sm.tbl[1][b1][nb];
  sum += (double)sm.tbl[2][b2][nb];
  sum += (double)sm.tbl[3][b3][nb];
  return (float)sum;
}

// Candidate buffer flush. Entries [0, n_keys) are keys kept by the previous flush; the entries appended since are
// keys (generic queries, scored in pass 2) or, for pure disjunctions (`raw`), unscored (tf word << 32 | doc) pairs:
// pass 2 only tests the tf-pattern bound, the exact scores are computed here, one entry per thread, so the norm
// loads of a whole buffer overlap instead of stalling one warp at a time inside pass 2. Then sort, keep the best
// top_k, publish the k-th key as the query's threshold.
__device__ __forceinline__ void compact_candidates_v2(const StreamLaunch& L, StreamSmem& sm, const uint8_t* norms0, bool raw,
                                                      bool has_after, uint64_t after_key, int top_k, uint64_t* g_theta) {
  __syncthreads();
  int n = sm.cand_count;
  if (n > kCand) n = kCand;
  if (raw) {
    // score, then re-append only the entries that beat theta: the sort below usually sees a few hundred keys
    const unsigned long long theta = sm.theta;
    const int n_keys = sm.n_keys;
    constexpr int kPer = (kCand + kThreads - 1) / kThreads;
    uint64_t mine[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = n_keys + (int)threadIdx.x + j * kThreads;
      uint64_t key = 0ull;
      if (i < n) {
        const uint64_t e = sm.cand[i];
        const int32_t doc = (int32_t)(uint32_t)e;
        key = make_key(score_disjunction(L, sm, norms0, doc, (uint32_t)(e >> 32)), doc);
        if (!(key > theta) || (has_after && !(key < after_key))) key = 0ull;   // a real key is never 0 (low word = ~doc)
      }
      mine[j] = key;
    }
    __syncthreads();
    if (threadIdx.x == 0) sm.cand_count = n_keys;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPer; ++j)
      if (mine[j]) sm.cand[atomicAdd(&sm.cand_count, 1)] = mine[j];
    __syncthreads();
    n = sm.cand_count;
    if (n < top_k) {   // fewer than top_k keys in all: nothing to drop, no k-th key to publish, and the slice merge sorts
      if (threadIdx.x == 0) {
        sm.n_keys = n;
        const unsigned long long g = *(volatile unsigned long long*)g_theta;
        if (g > sm.theta) sm.theta = g;
      }
      __syncthreads();
      return;
    }
  }
  int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + threadIdx.x; i < m; i += blockDim.x) sm.cand[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(sm.cand, m);
  if (threadIdx.x == 0) {
    int keep = n < top_k ? n : top_k;
    sm.cand_count = keep;
    sm.n_keys = keep;
    if (keep == top_k) {
      unsigned long long kth = sm.cand[top_k - 1];
      unsigned long long old = atomicMax((unsigned long long*)g_theta, kth);
      unsigned long long t = old > kth ? old : kth;
      if (t > sm.theta) sm.theta = t;
    } else {
      unsigned long long g = *(volatile unsigned long long*)g_theta;
      if (g > sm.theta) sm.theta = g;
    }
  }
  __syncthreads();
}

// kSimple: every query of the launch is a pure disjunction of scoring term clauses over one text field, no deletes
// (the host splits the work list): only that instantiation carries the tf-pattern bound, deferred scoring, MAXSCORE,
// tf planes and the sparse mode; the other one carries the generic clause evaluation.
template <bool kSimple>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) posting_stream_kernel(const __grid_constant__ StreamLaunch L) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  StreamSmem& sm = *reinterpret_cast<StreamSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int wi = blockIdx.x;
  if (wi >= L.n_work) return;
  const int qi = L.work_query[wi];
  // work_slice: slice | flags << 24. Flag 1 = warm-up item: only the first kWarmGran granules of slice 0, its own output
  // list (index n_slices - 1), scheduled before every other item so that the query's other work items start with a
  // threshold; flag 2 = the slice-0 item of such a query: starts behind those granules.
  const int slice_raw = L.work_slice[wi];
  const int slice = slice_raw & 0xffffff;
  const int wflags = slice_raw >> 24;
  const long long t_start = L.mode_stats ? clock64() : 0ll;

  // every thread reads the three query fields the loads below depend on straight from global memory (one broadcast
  // transaction per warp), so the clause / granule-bound loads do not wait for thread 0's part of the set-up
  const int ncl = L.queries[qi].n_clauses, cbeg = L.queries[qi].clause_begin, n_term = L.queries[qi].n_term;
  if (tid == 32) sm.hits0 = *(volatile unsigned long long*)&L.total_hits[qi];
  if (tid == 0) {
    sm.q = L.queries[qi];
    sm.cand_count = 0;
    sm.n_keys = 0;
    sm.theta = *(volatile unsigned long long*)&L.theta[qi];
    for (int j = 0; j < kPoolSparse; ++j) mbar_init(&sm.full_bar[j], 1);
    mbar_init(&sm.plane_bar[0], 1);
    mbar_init(&sm.plane_bar[1], 1);
    mbar_init(&sm.tab_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    // the query's tables (exact BM25 floats tbl[slot][tf][norm byte], bound per tf pattern ubt[]) were computed once
    // per batch by query_tables_kernel: one TMA copy brings both in while the rest of the set-up runs
    constexpr uint32_t kBytes = (uint32_t)kQTabFloats * 4u;
    const unsigned char* src = reinterpret_cast<const unsigned char*>(L.qtables + (size_t)qi * kQTabFloats);
    unsigned char* dst = reinterpret_cast<unsigned char*>(&sm.tbl[0][0][0]);
    mbar_arrive_expect_tx(&sm.tab_bar, kBytes);
    for (uint32_t o = 0; o < kBytes; o += 4096u) bulk_g2s(dst + o, src + o, min(4096u, kBytes - o), &sm.tab_bar);
  }
  if (tid < ncl) sm.cl[tid] = L.clauses[cbeg + tid];
  for (int i = tid; i < kW / 4; i += kThreads) reinterpret_cast<uint4*>(sm.slots)[i] = make_uint4(0u, 0u, 0u, 0u);
  // granule bounds of the slice (every list; lists served from their plane get their column cleared below)
  const int gran_per_slice = L.slice_docs >> kLogGran;           // 512
  const int g_first = slice * gran_per_slice;
  const int g_count = min(gran_per_slice, L.n_gran - g_first);     // granules of this slice
  const int g_lo = (wflags & 2) ? min(g_count, kWarmGran) : 0;     // granules [g_lo, g_hi) are this work item's
  const int g_hi = (wflags & 1) ? min(g_count, kWarmGran) : g_count;
#pragma unroll
  for (int t = 0; t < kT; ++t) {
    const uint32_t* p = L.gbounds + ((size_t)qi * kT + t) * (L.n_gran + 1) + g_first;
    for (int g = tid; g <= gran_per_slice; g += kThreads)
      reinterpret_cast<uint32_t*>(&sm.gb4[g])[t] = (t < n_term) ? p[min(g, g_count)] : 0u;
  }
  if (tid < kT) { sm.s_r_begin[tid] = 0; sm.s_r_end[tid] = 0; sm.s_n_chunks[tid] = 0; sm.s_issued[tid] = 0; sm.s_scoring[tid] = 0;
                  sm.s_gdocs[tid] = nullptr; sm.s_gf8[tid] = nullptr; sm.s_field[tid] = 0; sm.s_clause[tid] = 0;
                  sm.s_ring_base[tid] = 0; sm.s_ring_nch[tid] = 2; sm.s_plane[tid] = nullptr; }
  __syncthreads();
  // ---- MAXSCORE split (pure term disjunctions, once the query has collected more than totalHitsThreshold hits):
  // the lists whose list-wide score bounds sum (in double, ascending) to less than theta.score are non-essential --
  // a doc found only in them cannot beat theta. They never own a doc; the owners of the essential lists still see
  // their exact tf: from the list's dense tf plane when it has one (window mode: TMA copy per window; sparse mode:
  // byte gathers), else from its postings (scattered in window mode and cleared in pass 3, searched in sparse mode).
  // Rank-safe; docs matching only non-essential lists are not counted, so totalHits becomes a lower bound (relation
  // GREATER_THAN_OR_EQUAL_TO). Then the sweep mode of the work item (DESIGN.md 4.1) is chosen.
  if (tid == 0) {
    uint32_t ne = 0;
    const DevQuery& q = sm.q;
    const bool simple_q = kSimple;
    if (simple_q && sm.theta != 0ull && L.threshold < (int64_t)INT32_MAX &&
        (int64_t)sm.hits0 > L.threshold) {
      const float theta_s = key_score(sm.theta);
      float ub[kT]; int ord[kT]; int n = 0;
      for (int i = 0; i < q.n_clauses; ++i)
        if (sm.cl[i].kind == NRTGPU_TERM) { ub[sm.cl[i].slot] = sm.cl[i].ub; ord[n] = sm.cl[i].slot; ++n; }
      for (int a = 1; a < n; ++a) { int x = ord[a], b = a - 1; while (b >= 0 && ub[ord[b]] > ub[x]) { ord[b + 1] = ord[b]; --b; } ord[b + 1] = x; }
      double pre = 0.0;
      for (int a = 0; a < n; ++a) {
        const double s2 = pre + (double)ub[ord[a]];
        if (!((float)s2 < theta_s)) break;
        pre = s2; ne |= 1u << ord[a];
      }
    }
    sm.ne_mask = ne;
    if (ne) L.pruned[qi] = 1;
    // the densest non-essential list that has a dense tf plane is not streamed as postings at all: each window's
    // bytes of the plane are copied in by the TMA and the owners of pass 2 look their doc up (two ring-less lists
    // would not leave enough pool for the plane buffers, so queries of up to three terms only)
    // Sparse mode: when every list is either short in this slice or a non-essential list with a plane, the window
    // array is not needed at all -- the short lists are merged by binary search of each other's ring segments and the
    // plane bytes are read straight from L2. Windows then span as many granules as the rings hold (often the slice).
    int sp = 0; uint32_t pm = 0;
    if (simple_q) {
      sp = 1;
      for (int i = 0; i < q.n_clauses && sp; ++i) {
        const DevClause& c = sm.cl[i];
        if (c.kind != NRTGPU_TERM) continue;
        if (((ne >> c.slot) & 1u) && c.plane >= 0 && L.ix.dense_tf != nullptr) { pm |= 1u << c.slot; continue; }
        const uint32_t n_slice = reinterpret_cast<const uint32_t*>(&sm.gb4[g_hi])[c.slot] -
                                 reinterpret_cast<const uint32_t*>(&sm.gb4[g_lo])[c.slot];
        if (n_slice > (uint32_t)(ne ? kSparseCap : kSparseCapAll)) sp = 0;
      }
      if (!sp) pm = 0;
    }
    sm.sparse = sp; sm.pserve_mask = pm;
    int ps = -1;
    if (!sp && ne && q.n_term <= 3 && L.ix.dense_tf != nullptr) {
      float best = INFINITY;
      for (int i = 0; i < q.n_clauses; ++i) {
        const DevClause& c = sm.cl[i];
        if (c.kind == NRTGPU_TERM && ((ne >> c.slot) & 1u) && c.plane >= 0 && c.ub < best) { best = c.ub; ps = c.slot; }
      }
    }
    sm.plane_slot = ps;
  }
  __syncthreads();
  const uint32_t ne_mask = kSimple ? sm.ne_mask : 0u;
  const int pslot = kSimple ? sm.plane_slot : -1;
  const bool sparse = kSimple && sm.sparse != 0;
  const uint32_t pserve_mask = kSimple ? sm.pserve_mask : 0u;
  if (tid < ncl && sm.cl[tid].kind == NRTGPU_TERM) {
    const int s = sm.cl[tid].slot;
    const bool served = s == pslot || ((pserve_mask >> s) & 1u);   // plane-served lists are not streamed: no postings
    const int64_t g0 = sm.cl[tid].post_base + (served ? 0u : reinterpret_cast<const uint32_t*>(&sm.gb4[g_lo])[s]),
                  g1 = sm.cl[tid].post_base + (served ? 0u : reinterpret_cast<const uint32_t*>(&sm.gb4[g_hi])[s]);
    const int64_t base_g = (g0 >> kLogCH) << kLogCH;
    sm.s_r_begin[s] = (int32_t)(g0 - base_g);
    sm.s_r_end[s] = (int32_t)(g1 - base_g);
    sm.s_n_chunks[s] = (g1 > g0) ? (int32_t)((g1 - base_g + kCH - 1) >> kLogCH) : 0;
    sm.s_gdocs[s] = L.ix.post_docs + base_g;
    sm.s_gf8[s] = L.ix.post_f8 + base_g;
    sm.s_scoring[s] = sm.cl[tid].scoring != 0;
    sm.s_field[s] = sm.cl[tid].field;
    sm.s_clause[s] = tid;
    sm.s_plane[s] = (sm.cl[tid].plane >= 0 && L.ix.dense_tf != nullptr)
                        ? L.ix.dense_tf + (size_t)sm.cl[tid].plane * (size_t)L.ix.dense_stride : nullptr;
  }
  if (pslot >= 0 || pserve_mask != 0u) {   // plane-served lists have no postings in the rings: empty column
#pragma unroll
    for (int t = 0; t < kT; ++t)
      if (t == pslot || ((pserve_mask >> t) & 1u))
        for (int g = tid; g <= gran_per_slice; g += kThreads) reinterpret_cast<uint32_t*>(&sm.gb4[g])[t] = 0u;
  }
  __syncthreads();
  if (tid == 0) {
    // split the ring pool: every list gets at least one granule's worth (kMinNCH chunks, or the whole
    // list if shorter); the list with the most chunks still to stream per ring chunk is doubled while
    // the pool allows (dense lists get long rings = deep TMA prefetch)
    int nch[kT], used = 0;
    // (window mode with a plane: the tail of the pool holds the plane buffers; sparse mode: the pool runs on over the window array)
    const int pool_lim = sparse ? kPoolSparse : (pslot >= 0 ? kPool - kPlaneChunks : kPool);
    for (int t = 0; t < kT; ++t) {
      nch[t] = 0;
      if (t < n_term && t != pslot && !((pserve_mask >> t) & 1u)) { nch[t] = 2; while (nch[t] < kMinNCH && nch[t] < sm.s_n_chunks[t] + 1) nch[t] *= 2; }
      used += nch[t];
    }
    for (;;) {
      int best = -1; float best_ratio = 0.5f;
      for (int t = 0; t < n_term; ++t) {
        if (nch[t] == 0 || nch[t] >= kMaxNCH || used + nch[t] > pool_lim) continue;
        float ratio = (float)sm.s_n_chunks[t] / (float)nch[t];
        if (ratio > best_ratio) { best_ratio = ratio; best = t; }
      }
      if (best < 0) break;
      used += nch[best]; nch[best] *= 2;
    }
    int base = 0;
    for (int t = 0; t < kT; ++t) { sm.s_ring_base[t] = base; sm.s_ring_nch[t] = nch[t] ? nch[t] : 2; base += nch[t]; }
  }
  __syncthreads();

  // tf bytes of ring chunk s live at pf8 + s * kCH
  uint8_t* const pf8 = sparse ? reinterpret_cast<uint8_t*>(sm.slots) + kSparseF8Off : sm.pool_f8;
  static_assert(offsetof(StreamSmem, slots) == offsetof(StreamSmem, pool_docs) + sizeof(int32_t) * kPool * kCH &&
                offsetof(StreamSmem, pool_f8) == offsetof(StreamSmem, slots) + sizeof(uint32_t) * kW, "pool_docs / slots / pool_f8 contiguous");
  // ---- CTA-uniform per-slot registers
  int32_t r_cur[kT], rbase[kT], rmask[kT], issued[kT], waited[kT];
#pragma unroll
  for (int t = 0; t < kT; ++t) {
    r_cur[t] = sm.s_r_begin[t];
    rbase[t] = sm.s_ring_base[t] << kLogCH;
    rmask[t] = (sm.s_ring_nch[t] << kLogCH) - 1;
    issued[t] = 0;   // chunks handed to the TMA so far (tracked by warp 0, the issuing warp)
    waited[t] = 0;   // chunks whose arrival this warp has already observed
  }
  // the window table: from granule g the window runs to nextg[g] = the farthest granule (<= g + kWinGran) whose
  // postings fit every ring with one chunk of alignment slack. One granule always fits (<= kGran postings).
  // (sparse mode has no window array, so only the rings bound the run)
  for (int g = g_lo + tid; g < g_hi; g += kThreads) {
    const uint4 a = sm.gb4[g];
    auto fits = [&](int g1) {
      const uint4 b = sm.gb4[g1];
      return (int32_t)(b.x - a.x) <= rmask[0] + 1 - kCH && (int32_t)(b.y - a.y) <= rmask[1] + 1 - kCH &&
             (int32_t)(b.z - a.z) <= rmask[2] + 1 - kCH && (int32_t)(b.w - a.w) <= rmask[3] + 1 - kCH;
    };
    int hi = sparse ? g_hi : min(g_hi, g + kWinGran);
    int lo = g + 1;                     // always accepted
    if (hi > lo && !fits(hi)) {         // posting counts grow with g1: binary search the last run that fits
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (fits(mid)) lo = mid; else hi = mid; }
      hi = lo;
    }
    sm.nextg[g] = (uint16_t)hi;
  }
  // warp 0 fills every free ring slot, one chunk per lane (each chunk: expect_tx + two bulk copies on its mbarrier)
  auto issue_chunks = [&]() {
    if (tid >= 32) return;
#pragma unroll
    for (int t = 0; t < kT; ++t) {
      const int nchm = rmask[t] >> kLogCH;
      const int lim = min(sm.s_n_chunks[t], (r_cur[t] >> kLogCH) + nchm + 1);
      for (int j = issued[t] + lane; j < lim; j += 32) {
        const int slot = (rbase[t] >> kLogCH) + (j & nchm);
        uint64_t* bar = &sm.full_bar[slot];
        mbar_arrive_expect_tx(bar, kChunkBytes);
        bulk_g2s(&sm.pool_docs[slot << kLogCH], sm.s_gdocs[t] + ((size_t)j << kLogCH), kCH * 4, bar);
        bulk_g2s(pf8 + (slot << kLogCH), sm.s_gf8[t] + ((size_t)j << kLogCH), kCH, bar);
      }
      issued[t] = max(issued[t], lim);
    }
  };
  issue_chunks();

  static_assert(offsetof(StreamSmem, ubt) == offsetof(StreamSmem, tbl) + sizeof(float) * kT * (kTfTab + 1) * 256, "tbl/ubt adjacent");
  const bool simple = kSimple;
  if (lane == 0) mbar_wait(&sm.tab_bar, 0);
  __syncthreads();

  const int32_t slice_base = slice * L.slice_docs;
  int32_t slice_end = slice_base + L.slice_docs;
  if (slice_end > L.ix.n_docs || slice_end < slice_base) slice_end = L.ix.n_docs;
  const bool dense = !kSimple && sm.q.dense_driver != 0;
  const bool has_after = sm.q.has_after != 0;
  const uint64_t after_key = sm.q.after_key;
  const uint32_t driver_mask = sm.q.driver_mask & ~ne_mask;            // non-essential lists never own a doc
  const bool has_non_driver = sm.q.has_non_driver != 0 || ne_mask != 0;  // ... pass 3 clears their words
  const uint8_t* norms0 = (sm.q.single_field >= 0) ? L.ix.norms[sm.q.single_field] : nullptr;
  uint32_t scoring_bits = 0;
#pragma unroll
  for (int t = 0; t < kT; ++t) scoring_bits |= (sm.s_scoring[t] ? 1u : 0u) << t;
  // word bytes of the driver slots below each slot (ownership test)
  const uint32_t drv_bytes = ((driver_mask & 1u) ? 0xffu : 0u) | ((driver_mask & 2u) ? 0xff00u : 0u) |
                             ((driver_mask & 4u) ? 0xff0000u : 0u) | ((driver_mask & 8u) ? 0xff000000u : 0u);
  unsigned int my_hits = 0;
  unsigned char* slot_bytes = reinterpret_cast<unsigned char*>(sm.slots);

  int g0 = g_lo;   // next granule of the slice
  if (n_term > 0 && ne_mask == ((1u << n_term) - 1u)) g0 = g_hi;   // every list is non-essential: skip the slice
  // ---- tf plane of the plane-served list: window n's bytes live in buffer n & 1 (filled two windows ahead)
  uint8_t* const pb = reinterpret_cast<uint8_t*>(sm.pool_docs + (kPool - kPlaneChunks) * kCH);
  const uint8_t* const psrc =
      pslot >= 0 ? L.ix.dense_tf + (size_t)sm.cl[sm.s_clause[pslot]].plane * (size_t)L.ix.dense_stride : nullptr;
  const uint32_t pshift = pslot >= 0 ? 8u * (uint32_t)pslot : 0u;
  auto issue_plane = [&](int n, int ga, int gb) {   // one thread: granules [ga, gb) of the slice
    const int32_t wb = slice_base + (ga << kLogGran);
    const int32_t we = min(slice_end, slice_base + (gb << kLogGran));
    const uint32_t bytes = (uint32_t)(we - wb + 15) & ~15u;   // the plane is padded past n_docs
    uint64_t* bar = &sm.plane_bar[n & 1];
    mbar_arrive_expect_tx(bar, bytes);
    for (uint32_t o = 0; o < bytes; o += 4096u)
      bulk_g2s(pb + (n & 1) * kW + o, psrc + wb + o, min(4096u, bytes - o), bar);
  };
  if (pslot >= 0 && tid == 0 && g0 < g_hi) {
    const int ga = sm.nextg[g0];
    issue_plane(0, g0, ga);
    if (ga < g_hi) issue_plane(1, ga, sm.nextg[ga]);
  }
  unsigned long long dbg_postings = 0;   // driver postings visited (NRTGPU_DEBUG_MODES)
  const long long t_loop = L.mode_stats ? clock64() : 0ll;
  unsigned long long dbg_windows = 0;
  int wn = 0;   // window counter (skipped windows count too: each has its plane copy)
  while (g0 < g_hi) {
    // ---------------- window = the longest run of granules (<= kWinGran) whose postings fit every ring
    const int g1 = sm.nextg[g0];
    int32_t cnt[kT];
    const uint4 gb_w = sm.gb4[g0];   // postings of every list below the window's first granule
    {
      const uint4 b = sm.gb4[g1];
      cnt[0] = (int32_t)(b.x - gb_w.x); cnt[1] = (int32_t)(b.y - gb_w.y); cnt[2] = (int32_t)(b.z - gb_w.z); cnt[3] = (int32_t)(b.w - gb_w.w);
    }
    const int32_t wbase = slice_base + (g0 << kLogGran);
    const int32_t wend = min(slice_end, slice_base + (g1 << kLogGran));
    g0 = g1;
    // ---------------- residency: every warp waits for the chunks that hold [r_cur, r_cur + cnt)
    // (each chunk is awaited once per warp: `waited` remembers how far this warp has looked; lanes take one chunk each)
    {
      int need[kT], total = 0;
#pragma unroll
      for (int t = 0; t < kT; ++t) {
        const int jl1 = (cnt[t] > 0) ? ((r_cur[t] + cnt[t] - 1) >> kLogCH) + 1 : 0;   // one past the last chunk needed
        need[t] = max(jl1 - waited[t], 0);
        total += need[t];
      }
      if (total > 0) {
        for (int l = lane; l < total; l += 32) {
          int t = 0, k = l;
          if (k >= need[0]) { k -= need[0]; t = 1;
            if (k >= need[1]) { k -= need[1]; t = 2;
              if (k >= need[2]) { k -= need[2]; t = 3; } } }
          const int w0 = t == 0 ? waited[0] : t == 1 ? waited[1] : t == 2 ? waited[2] : waited[3];
          const int nch = sm.s_ring_nch[t];
          const int j = w0 + k;
          mbar_wait(&sm.full_bar[sm.s_ring_base[t] + (j & (nch - 1))], (j >> (31 - __clz(nch))) & 1);
        }
#pragma unroll
        for (int t = 0; t < kT; ++t) waited[t] += need[t];
        __syncwarp();
      }
    }

    if (pslot >= 0) {
      if (lane == 0) mbar_wait(&sm.plane_bar[wn & 1], (wn >> 1) & 1);
      __syncwarp();
    }
    auto next_plane = [&]() {   // after the window's last barrier: buffer wn & 1 is free for window wn + 2
      if (pslot >= 0 && tid == 0 && g1 < g_hi) {
        const int g2 = sm.nextg[g1];
        if (g2 < g_hi) issue_plane(wn + 2, g2, sm.nextg[g2]);
      }
      ++wn;
    };
    {
      int32_t ess = 0;
#pragma unroll
      for (int t = 0; t < kT; ++t) if (!((ne_mask >> t) & 1u)) ess |= cnt[t];
      if (!dense && ess == 0) {   // no posting of an essential list in these granules: just advance the streams
#pragma unroll
        for (int t = 0; t < kT; ++t) r_cur[t] += cnt[t];
        __syncthreads();   // every warp has seen these chunks land (mbarrier phases only tell odd from even: a ring
        issue_chunks();    // slot is re-armed only after ALL warps observed its previous phase)
        next_plane();
        continue;
      }
    }

    if (L.mode_stats) {
      ++dbg_windows;
#pragma unroll
      for (int t = 0; t < kT; ++t) if ((driver_mask >> t) & 1u) dbg_postings += (unsigned long long)cnt[t];
    }
    // the window's postings are dealt round-robin over the threads ACROSS the clauses (clause t starts where
    // clause t-1 stopped), so short lists do not pile onto the first warps
    int32_t rot[kT];
    rot[0] = 0;
#pragma unroll
    for (int t = 1; t < kT; ++t) rot[t] = (rot[t - 1] + cnt[t - 1]) & (kThreads - 1);
    if (sparse) {
      // ---------------- sparse mode: one pass, no window array. Every posting of a driver list looks its doc up in
      // the other streamed lists' ring segments (binary search, narrowed to the doc's own 1024-doc granule by the
      // granule bounds); the lowest driver list that holds the doc owns it. A thread works on TWO postings at a time
      // (a CTA stride apart): their plane gathers and search chains are independent and overlap.
      int32_t it[kT];
#pragma unroll
      for (int t = 0; t < kT; ++t) it[t] = (tid - rot[t]) & (kThreads - 1);
      int npend = 0;
      uint64_t pk0 = 0, pk1 = 0;
      auto push = [&](uint64_t raw) {
        const int p = atomicAdd(&sm.cand_count, 1);
        if (p < kCand) sm.cand[p] = raw;
        else { if (npend == 0) pk0 = raw; else pk1 = raw; ++npend; }
      };
      for (;;) {
        const unsigned long long theta = sm.theta;
        const float theta_s = theta ? key_score(theta) : -INFINITY;
        if (npend) {   // parked by the last flush: append again
          const int n = npend; const uint64_t a = pk0, b = pk1;
          npend = 0;
          push(a);
          if (n > 1) push(b);
        }
        if (!npend) {
#pragma unroll
          for (int t = 0; t < kT; ++t) {
            if (t >= n_term || npend) break;
            if (!((driver_mask >> t) & 1u)) continue;
            const int32_t* rd = sm.pool_docs + rbase[t];
            const uint8_t* rf = pf8 + rbase[t];
            int32_t i = it[t];
#pragma unroll 1
            for (; i < cnt[t]; i += 2 * kThreads) {
              const bool hasB = i + kThreads < cnt[t];
              const int idxA = (r_cur[t] + i) & rmask[t], idxB = (r_cur[t] + i + kThreads) & rmask[t];
              const int32_t docA = rd[idxA], docB = hasB ? rd[idxB] : docA;
              uint32_t vA = (uint32_t)rf[idxA] << (8 * t), vB = (uint32_t)rf[idxB] << (8 * t);
#pragma unroll
              for (int u = 0; u < kT; ++u)
                if ((pserve_mask >> u) & 1u) {
                  const uint8_t* pl = sm.s_plane[u];
                  const uint32_t a = __ldg(pl + docA), b = __ldg(pl + docB);
                  vA |= a << (8 * u); vB |= b << (8 * u);
                }
              const int gA = (docA - slice_base) >> kLogGran, gB = (docB - slice_base) >> kLogGran;
              bool ownA = true, ownB = hasB;
#pragma unroll
              for (int u = 0; u < kT; ++u) {
                if (u == t || u >= n_term || cnt[u] == 0) continue;
                const int32_t* ud = sm.pool_docs + rbase[u];
                const uint32_t w0 = reinterpret_cast<const uint32_t*>(&gb_w)[u];
                int32_t loA = (int32_t)(reinterpret_cast<const uint32_t*>(&sm.gb4[gA])[u] - w0);
                int32_t loB = (int32_t)(reinterpret_cast<const uint32_t*>(&sm.gb4[gB])[u] - w0);
                const int32_t endA = (int32_t)(reinterpret_cast<const uint32_t*>(&sm.gb4[gA + 1])[u] - w0);
                const int32_t endB = (int32_t)(reinterpret_cast<const uint32_t*>(&sm.gb4[gB + 1])[u] - w0);
                int32_t hiA = endA, hiB = endB;
                while ((loA < hiA) | (loB < hiB)) {
                  const int32_t midA = (loA + hiA) >> 1, midB = (loB + hiB) >> 1;
                  const int32_t dA = ud[(r_cur[u] + midA) & rmask[u]], dB = ud[(r_cur[u] + midB) & rmask[u]];
                  if (loA < hiA) { if (dA < docA) loA = midA + 1; else hiA = midA; }
                  if (loB < hiB) { if (dB < docB) loB = midB + 1; else hiB = midB; }
                }
                const int uA = (r_cur[u] + loA) & rmask[u], uB = (r_cur[u] + loB) & rmask[u];
                const bool lower_driver = u < t && ((driver_mask >> u) & 1u);
                if (loA < endA && ud[uA] == docA) {
                  if (lower_driver) ownA = false;   // counted and emitted by list u's thread
                  else vA |= (uint32_t)pf8[rbase[u] + uA] << (8 * u);
                }
                if (loB < endB && ud[uB] == docB) {
                  if (lower_driver) ownB = false;
                  else vB |= (uint32_t)pf8[rbase[u] + uB] << (8 * u);
                }
              }
              if (ownA) {
                ++my_hits;
                if (!(sm.ubt[__dp4a(__vminu4(vA, 0x05050505u), 0xD8240601u, 0u)] < theta_s)) push(((uint64_t)vA << 32) | (uint32_t)docA);
              }
              if (ownB) {
                ++my_hits;
                if (!(sm.ubt[__dp4a(__vminu4(vB, 0x05050505u), 0xD8240601u, 0u)] < theta_s)) push(((uint64_t)vB << 32) | (uint32_t)docB);
              }
              if (npend) { i += 2 * kThreads; break; }
            }
            it[t] = i;
          }
        }
        __syncthreads();
        if (sm.cand_count <= kCand) break;
        compact_candidates_v2(L, sm, norms0, true, has_after, after_key, L.top_k, &L.theta[qi]);
      }
#pragma unroll
      for (int t = 0; t < kT; ++t) r_cur[t] += cnt[t];
      issue_chunks();
      next_plane();
      continue;
    }
    // ---------------- pass 1: scatter tf bytes
#pragma unroll
    for (int t = 0; t < kT; ++t) {
      if (t >= n_term) break;
      const bool scoring = (scoring_bits >> t) & 1u;
      const int32_t* rd = sm.pool_docs + rbase[t];
      const uint8_t* rf = sm.pool_f8 + rbase[t];
      unsigned char* sb = slot_bytes + t - 4 * wbase;
#pragma unroll 1
      for (int32_t i = (tid - rot[t]) & (kThreads - 1); i < cnt[t]; i += kThreads) {   // a few postings per thread
        const int idx = (r_cur[t] + i) & rmask[t];
        sb[4 * rd[idx]] = scoring ? rf[idx] : (unsigned char)1;
      }
    }
    __syncthreads();
    // ---------------- pass 2: owners emit. No barrier inside: a thread whose candidate does not fit the
    // buffer parks it (pending) and stops; the CTA then compacts and the parked threads resume.
    {
      int32_t it[kT];
#pragma unroll
      for (int t = 0; t < kT; ++t) it[t] = (tid - rot[t]) & (kThreads - 1);
      const uint8_t* const pbw = pb + (wn & 1) * kW - wbase;   // plane byte of doc d: pbw[d]
      int32_t idense = tid;
      bool pending = false;
      uint64_t pkey = 0;
      for (;;) {
        const unsigned long long theta = sm.theta;
        const float theta_s = theta ? key_score(theta) : -INFINITY;
        if (pending) {
          pending = false;
          if (simple || pkey > theta) {
            const int p = atomicAdd(&sm.cand_count, 1);
            if (p < kCand) sm.cand[p] = pkey; else pending = true;
          }
        }
        if (!pending) {
          if (!dense) {
#pragma unroll
            for (int t = 0; t < kT; ++t) {
              if (t >= n_term || pending) break;
              if (!((driver_mask >> t) & 1u)) continue;
              const uint32_t own = 0xffu << (8 * t), bel = drv_bytes & ((1u << (8 * t)) - 1u);
              const int32_t* rd = sm.pool_docs + rbase[t];
              uint32_t* sl = sm.slots - wbase;
              int32_t i = it[t];
              if (simple) {
#pragma unroll 1
                for (; i < cnt[t]; i += kThreads) {
                  const int32_t doc = rd[(r_cur[t] + i) & rmask[t]];
                  const uint32_t v = sl[doc];
                  if ((v & bel) != 0 || (v & own) == 0) continue;   // a lower driver slot owns this doc
                  sl[doc] = 0u;
                  ++my_hits;
                  const uint32_t vv = pslot >= 0 ? (v | ((uint32_t)pbw[doc] << pshift)) : v;   // + the plane-served list's tf
                  const uint32_t ui = __dp4a(__vminu4(vv, 0x05050505u), 0xD8240601u, 0u);   // sum min(tf_s, 5) * 6^s
                  if (sm.ubt[ui] < theta_s) continue;               // cannot reach the top-k
                  const uint64_t raw = ((uint64_t)vv << 32) | (uint32_t)doc;   // scored at the next flush
                  const int p = atomicAdd(&sm.cand_count, 1);
                  if (p < kCand) sm.cand[p] = raw;
                  else { pending = true; pkey = raw; i += kThreads; break; }
                }
              } else {
                for (; i < cnt[t]; i += kThreads) {
                  const int32_t doc = rd[(r_cur[t] + i) & rmask[t]];
                  const uint32_t v = sl[doc];
                  if ((v & bel) != 0 || (v & own) == 0) continue;
                  sl[doc] = 0u;
                  float score;
                  if (!evaluate_doc_generic(L, sm, doc, v, &score)) continue;
                  ++my_hits;
                  const uint64_t key = make_key(score, doc);
                  if (key > theta && (!has_after || key < after_key)) {
                    const int p = atomicAdd(&sm.cand_count, 1);
                    if (p < kCand) sm.cand[p] = key;
                    else { pending = true; pkey = key; i += kThreads; break; }
                  }
                }
              }
              it[t] = i;
            }
          } else {
            const int32_t wlen = wend - wbase;
            int32_t i = idense;
            for (; i < wlen; i += kThreads) {
              const uint32_t v = sm.slots[i];
              if (v) sm.slots[i] = 0u;
              float score;
              if (!evaluate_doc_generic(L, sm, wbase + i, v, &score)) continue;
              ++my_hits;
              const uint64_t key = make_key(score, wbase + i);
              if (key > theta && (!has_after || key < after_key)) {
                const int p = atomicAdd(&sm.cand_count, 1);
                if (p < kCand) sm.cand[p] = key;
                else { pending = true; pkey = key; i += kThreads; break; }
              }
            }
            idense = i;
          }
        }
        __syncthreads();
        if (sm.cand_count <= kCand) break;                 // nobody is parked
        compact_candidates_v2(L, sm, norms0, simple, has_after, after_key, L.top_k, &L.theta[qi]);  // raises theta, frees the buffer
      }
    }
    // ---------------- pass 3: clear the words pass 2 did not visit
    // (by posting when the non-driver lists are sparse here, else one 128-bit sweep over the window's words)
    if (!dense && has_non_driver) {
      int32_t nd = 0;
#pragma unroll
      for (int t = 0; t < kT; ++t) if (!((driver_mask >> t) & 1u)) nd += cnt[t];
      if (nd > 2 * kThreads) {
        uint4* s4 = reinterpret_cast<uint4*>(sm.slots);
        const int n4 = (wend - wbase + 3) >> 2;
        for (int i = tid; i < n4; i += kThreads) s4[i] = make_uint4(0u, 0u, 0u, 0u);
      } else if (nd > 0) {
#pragma unroll
        for (int t = 0; t < kT; ++t) {
          if (t >= n_term) break;
          if ((driver_mask >> t) & 1u) continue;
          for (int32_t i = tid; i < cnt[t]; i += kThreads)
            sm.slots[sm.pool_docs[rbase[t] + ((r_cur[t] + i) & rmask[t])] - wbase] = 0u;
        }
      }
      if (nd > 0) __syncthreads();
    }
    // ---------------- advance the streams, refill freed ring slots
#pragma unroll
    for (int t = 0; t < kT; ++t) r_cur[t] += cnt[t];
    issue_chunks();
    next_plane();
  }

  const long long t_flush = L.mode_stats ? clock64() : 0ll;
  // ---------------- finish the work item: the slice merge sorts, so only a full buffer needs ordering here
  __syncthreads();
  if (simple ? sm.cand_count > sm.n_keys : sm.cand_count > L.top_k)
    compact_candidates_v2(L, sm, norms0, simple, has_after, after_key, L.top_k, &L.theta[qi]);
  const int keep = min(sm.cand_count, L.top_k);
  const int out_list = (wflags & 1) ? L.n_slices - 1 : slice;
  uint64_t* out = L.slice_keys + ((size_t)qi * L.n_slices + out_list) * L.top_k;
  for (int i = tid; i < keep; i += kThreads) out[i] = sm.cand[i];
  if (tid == 0) L.slice_cnt[(size_t)qi * L.n_slices + out_list] = keep;
  for (int o = 16; o > 0; o >>= 1) my_hits += __shfl_xor_sync(0xffffffffu, my_hits, o);
  if (lane == 0 && my_hits) atomicAdd(&L.total_hits[qi], (unsigned long long)my_hits);
  if (L.mode_stats && tid == 0) {
    const int mode = sparse ? 2 : (ne_mask ? 1 : 0);
    atomicAdd(&L.mode_stats[2 * mode], (unsigned long long)(clock64() - t_start));
    atomicAdd(&L.mode_stats[2 * mode + 1], 1ull);
    atomicAdd(&L.mode_stats[6 + mode], dbg_postings);
    if (mode == 2) {
      atomicAdd(&L.mode_stats[9], (unsigned long long)(t_loop - t_start));
      atomicAdd(&L.mode_stats[10], (unsigned long long)(t_flush - t_loop));
      atomicAdd(&L.mode_stats[11], (unsigned long long)(clock64() - t_flush));
      atomicAdd(&L.mode_stats[12], dbg_windows);
    }
  }
}

// tbl[slot][tf][norm byte] and ubt[tf pattern] of every query, once per batch (the 20 work items of a query share them)
struct QTabLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  const uint8_t* field_min_norm;  // [n_fields] norm byte of the shortest field value present (tightest score bound)
  int32_t nq;
  float* qtables;
};

__global__ void __launch_bounds__(256) query_tables_kernel(QTabLaunch Q) {
  const int q = blockIdx.x;
  if (q >= Q.nq) return;
  __shared__ DevClause cl[kT];
  __shared__ int have[kT];
  const DevQuery dq = Q.queries[q];
  if (threadIdx.x < kT) have[threadIdx.x] = 0;
  __syncthreads();
  if ((int)threadIdx.x < dq.n_clauses) {
    const DevClause c = Q.clauses[dq.clause_begin + threadIdx.x];
    if (c.kind == NRTGPU_TERM && c.slot >= 0 && c.slot < kT) { cl[c.slot] = c; have[c.slot] = 1; }
  }
  __syncthreads();
  float* out = Q.qtables + (size_t)q * kQTabFloats;
  for (int i = threadIdx.x; i < kT * (kTfTab + 1) * 256; i += blockDim.x) {
    const int s = i / ((kTfTab + 1) * 256), tf = (i / 256) % (kTfTab + 1), nb = i & 255;
    float v = 0.0f;
    if (have[s] && tf > 0 && cl[s].scoring) v = bm25_score(cl[s].weight, (float)tf, __ldg(&Q.ix.caches[cl[s].field * 256 + nb]));
    out[i] = v;
  }
  // upper bounds per tf pattern (used by pure single-field disjunctions): the same double sum, each term at the
  // shortest field length present (largest score); tf >= 5 is bounded by the clause weight (limit tf -> inf)
  const uint32_t nbmin = (dq.single_field >= 0 && Q.field_min_norm) ? (uint32_t)Q.field_min_norm[dq.single_field] : 0u;
  float* ub = out + kT * (kTfTab + 1) * 256;
  for (int i = threadIdx.x; i < kUbt; i += blockDim.x) {
    const int c[kT] = {i % 6, (i / 6) % 6, (i / 36) % 6, i / 216};
    double sum = 0.0;
#pragma unroll
    for (int t = 0; t < kT; ++t) {
      float u = 0.0f;
      if (have[t] && c[t] > 0)
        u = (c[t] <= 4) ? bm25_score(cl[t].weight, (float)c[t], __ldg(&Q.ix.caches[cl[t].field * 256 + nbmin])) : cl[t].weight;
      sum += (double)u;
    }
    ub[i] = (float)sum;
  }
}

// postings of every (query, term slot) below each 2048-doc granule boundary (relative to the clause's list)
struct BoundsLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  int32_t nq, n_gran;
  uint32_t* gbounds;  // [nq][kT][n_gran+1]
};

__global__ void granule_bounds_kernel(BoundsLaunch B) {
  const int64_t per_q = (int64_t)kT * (B.n_gran + 1);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B.nq * per_q) return;
  const int q = (int)(i / per_q), s = (int)((i % per_q) / (B.n_gran + 1)), g = (int)(i % (B.n_gran + 1));
  const DevQuery dq = B.queries[q];
  uint32_t out = 0;
  for (int c = 0; c < dq.n_clauses; ++c) {
    const DevClause cl = B.clauses[dq.clause_begin + c];
    if (cl.kind != NRTGPU_TERM || cl.slot != s) continue;
    if (cl.gran_row >= 0) { out = __ldg(B.ix.gran_tab + (size_t)cl.gran_row * (B.n_gran + 1) + g); break; }   // index-time skip data
    const int64_t target64 = (int64_t)g << kLogGran;
    const int32_t target = target64 > (int64_t)B.ix.n_docs ? B.ix.n_docs : (int32_t)target64;
    const int32_t* docs = B.ix.post_docs + cl.post_base;
    int lo = 0, hi = cl.n_post;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(docs + mid) < target) lo = mid + 1; else hi = mid; }
    out = (uint32_t)lo;
  }
  B.gbounds[i] = out;
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
  const int64_t target64 = (int64_t)g << kLogGran;
  const int32_t target = target64 > (int64_t)G.n_docs ? G.n_docs : (int32_t)target64;
  const int32_t* docs = G.post_docs + G.row_off[r];
  int lo = 0, hi = G.row_n[r];
  while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(docs + mid) < target) lo = mid + 1; else hi = mid; }
  G.tab[i] = (uint32_t)lo;
}

}  // namespace v2
}  // namespace nrtgpu
