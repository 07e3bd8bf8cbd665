// posting_probe_kernel -- the batched BooleanQuery engine of round 2 for queries of <= 4 term clauses that a posting
// list can lead (DESIGN.md 4.1). It replaces, for a whole batch of queries, what Lucene does per query in
//   MaxScoreBulkScorer (pure disjunctions, essential / non-essential partition),
//   ConjunctionDISI / BlockMaxConjunctionBulkScorer (the rarest required list leads, the others are advanced to it),
//   ReqExclBulkScorer / ReqOptSumScorer (MUST_NOT and optional clauses looked up per candidate)
// behind IndexSearcher.search (reference src/main/java/com/yelp/nrtsearch/server/handler/SearchHandler.java:1412).
//
// Design (GPU-first, nothing like the per-document iterator chain of the reference):
//   * work item = (query, doc slice, part), claimed from an atomic queue by PERSISTENT CTAs (3 or 4 per SM): no per-CTA
//     launch cost; slice-major so that the CTAs resident together probe the same doc range of the dense tf planes in
//     L2; a heavy (query, slice) is split into 2..16 parts so that no item is a large share of the launch; warm-up
//     items first: a query sweeps the first 32K postings of its highest-bound list over the whole shard (lower-bound
//     scores, nothing output) and publishes a threshold before any of its other items runs;
//   * the kernel is data parallel over the DRIVER postings of the item: every thread takes postings of the lists
//     that lead (the essential lists of a disjunction, the rarest required list of a conjunction), and PROBES every
//     other list for the doc: a byte gather from the list's dense tf plane (index-time direct-address bytes, L2), or
//     a granule-narrowed binary search of the list's slice segment staged in shared memory by 1-D TMA bulk copies
//     (cp.async.bulk + mbarrier complete_tx). No window array, no scatter, no per-window barriers: one barrier per
//     round of kR * 256 postings, whose gathers are all in flight together;
//   * pure disjunctions: rank-safe tf-pattern bound test, then the exact Lucene floats (BM25Scorer expression, double
//     clause sums) a full warp at a time; only a key that beats the query's threshold enters the candidate buffer;
//     MAXSCORE partition from index-time list bounds and the query's running threshold theta (one global 64-bit word
//     per query, atomicMax: the device analogue of LazyMaxScoreAccumulator.java:21-70);
//   * exact totalHits without sweeping the densest list: hits = |L1| + sum over the other lists of the postings whose
//     doc is in no earlier list (inclusion by ownership), so in ScoreMode.COMPLETE a non-essential dense list with a
//     plane contributes its posting count and is never read;
//   * anything else (MUST / FILTER / MUST_NOT, ranges, several fields, deletes, minimumNumberShouldMatch): the
//     generic instantiation evaluates the clause tree per surviving driver posting (leap-frog: a doc missing a
//     required list is dropped after the probes, before any norm / doc-value gather).
// Results are bit-identical to the exhaustive oracle (tests/test_gpu_parity.py, tests/test_gpu_probe.py).
#pragma once
#include "query_eval.cuh"
#include "sort_kernel.cuh"
#include "collect_kernel.cuh"

namespace nrtgpu {
namespace v3 {

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
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// bit s set: byte s (term slot s) of a tf word is non-zero
__device__ __forceinline__ uint32_t presence4(uint32_t s) {
  return ((s & 0xffu) ? 1u : 0u) | ((s & 0xff00u) ? 2u : 0u) | ((s & 0xff0000u) ? 4u : 0u) | ((s & 0xff000000u) ? 8u : 0u);
}

// byte s 0xff where bit s of m is set (the inverse of presence4)
__device__ __forceinline__ uint32_t expand4(uint32_t m) {
  return ((m & 1u) ? 0xffu : 0u) | ((m & 2u) ? 0xff00u : 0u) | ((m & 4u) ? 0xff0000u : 0u) | ((m & 8u) ? 0xff000000u : 0u);
}

// profiling builds only (-DNRT_PROBE_KNOCK): parts of the kernel can be disabled at run time through ProbeLaunch::knock
#ifdef NRT_PROBE_KNOCK
#define NRT_KNOCK(bit) ((L.knock & (bit)) != 0)
#else
#define NRT_KNOCK(bit) false
#endif
// (kT, kCtasA, the granule, kMaxSliceGran, kWarmGran, kProbeMaxTopK and the work-item word: batch_plan.h)
// Two launch configurations of the same kernel: 3 CTAs / SM with an 8192-posting stage (80 registers; best for the
// MAXSCORE-pruned sweeps of TOP_SCORES, whose sparse leading lists want the larger stage) and 4 CTAs / SM with a
// 6656-posting stage (64 registers; best where every posting is visited: ScoreMode.COMPLETE and the generic clause
// evaluation, both latency bound on their gathers: 32 resident warps hide more of it than 24).
constexpr int kStageA = 8192;
constexpr int kCtasB = 4, kStageB = 6656;
constexpr int kThreads = 256;
constexpr int kAlign = 16;                  // staged segments start on 16-posting boundaries (TMA: 16-byte aligned tf bytes)
// padding postings behind the last list of the index image: a staged segment also ends on a kAlign-posting boundary of
// the global arrays (seg_n), so the segment of the last list can read up to kAlign - 1 postings past its end. 1024 is
// far more than that; the value keeps the image layout and nrtgpu_index_device_bytes unchanged.
constexpr int kPostingPad = 1024;
constexpr int kLongReserve = kT * (kGran + 2 * kAlign);   // one granule of every long list always fits
#ifndef NRT_PROBE_R
#define NRT_PROBE_R 2
#endif
constexpr int kR = NRT_PROBE_R;              // driver postings per thread per round (their gathers are in flight together)
constexpr int kCand = 1024;                  // candidate buffer entries
static_assert(kProbeMaxTopK == kCand / 2, "the probe kernel keeps top_k <= half its candidate buffer");
constexpr int kUbt = 4 * 4 * 4 * 4;          // tf-pattern bounds: min(tf, 3) per slot
static_assert(sizeof(DevProbeQuery::ubt) == kUbt * sizeof(float), "one bound per tf pattern");
constexpr int kWq = 32 * kR;                 // per-warp queue entries: the rounds drain it below 32 after their first push; once
                                             // the buffer is full, the kR - 1 pushes left in the round are not drained
constexpr int kProbeStats = 31;              // stats words per instantiation (ProbeLaunch::stats)
constexpr uint32_t kPiece = 8192;            // bytes per bulk copy
constexpr uint32_t kTfInexact = 0xFEu;       // tf byte of a plane probe whose 2-bit code saturated (tf >= 3): the exact byte is
                                             // fetched from the byte plane when the doc is scored (rare); >= 3 for the bound table

enum { kAbsent = 0, kLong = 1, kShort = 2, kPlane = 3, kGlobal = 4 };

struct ProbeLaunch {
  DevIndexView ix;
  const DevProbeQuery* pquery;   // [nq] per-query records (probe_query_kernel)
  const int32_t* work_query;
  const int32_t* work_slice;     // work-item word (batch_plan.h item_encode)
  const uint32_t* sbounds;       // [nq][kT][boundary_entries]: postings of the slot's list below every part boundary, the shard end, the
                                 // warm-up boundary, the end of the exact sweep warm-up
  unsigned int* work_counter;    // queue head
  unsigned long long* stats;     // optional [kProbeStats]: items, item cycles, runs, driver postings, flushes, staged runs, set-up
                                 // cycles, rounds, longest item, CTA busy (sum, max), warm-up items and cycles, flush, TMA wait and
                                 // flush_top_k cycles, queued entries, admitted keys; pure-disjunction items that started with no
                                 // threshold (count, cycles, in slice 0 / 1) and whose MAXSCORE roles went stale (count, cycles,
                                 // driver postings, postings of the lists that turned non-essential, in slice 0 / 1); exact sweep
                                 // warm-ups (count, driver postings, cycles)
  int32_t n_work, n_lists, n_slices, top_k;
  int32_t parts_max;             // result lists / boundary entries per slice (a heavy (query, slice) is split into up to this many items)
  int32_t slice_docs;            // multiple of kGran, <= kMaxSliceGran * kGran
  int32_t n_gran;
  int64_t threshold;             // INT32_MAX: ScoreMode.COMPLETE (exact counts)
  int32_t* pruned;
  uint64_t* theta;
  unsigned long long* total_hits;
  uint64_t* slice_keys;
  int32_t* slice_cnt;
  // deadline (SearchCutoffWrapper.java:164-174, checked at work-item boundaries = the reference's per-segment check):
  // the first work item of the run stamps clock0 with %globaltimer; an item claimed more than deadline_ns later is
  // skipped and its query flagged. terminateAfter (TerminateAfterWrapper.java:150-162): a query that has already
  // collected that many hits takes no further work items.
  long long deadline_ns;         // 0: no deadline; < 0: already expired
  unsigned long long* clock0;
  int32_t* timed_out;            // [nq]
  long long terminate_after;     // 0: none
  int32_t* terminated;           // [nq]
  // sort-by-field (generic instantiation): the key of a hit is (order-preserving code of its sort value, ~doc) instead
  // of (score, ~doc); see sort_kernel.cuh
  int32_t sort_kind, sort_reverse;
  const uint32_t* sort_codes;    // [n_docs] codes of the sort column (0 = doc without a value), or the 1-based ranks of a sort order
  const uint32_t* sort_missing_code;   // [1] code of the sort's missing value
  const AggLaunch* aggs;         // additional collectors (generic instantiation; device pointer, NULL: none)
  const unsigned long long* known_hits;   // optional [nq]: docs KNOWN to match (the longest list of a pure disjunction on a shard without
                                          // deletes): lets pruning start before that many hits were collected (totalHits > threshold is a fact)
  int32_t knock;                 // profiling only (NRTGPU_KNOCK): 1 no plane gathers, 2 no searches, 4 no appends, 8 no sweep
};

template <int kStageT>
struct alignas(128) ProbeSmemT {
  static constexpr int kStage = kStageT;             // postings of the searched lists resident in shared memory (5 B each)
  static constexpr int kShortMax = kStageT - kLongReserve;   // lists without skip data are staged whole, up to this many postings
  static_assert(kShortMax >= 1024, "stage too small");
  int32_t sdocs[kStageT];
  uint8_t sf8[kStageT];
  uint32_t gb[kT][kMaxSliceGran + 4];   // granule offsets of the slice for lists with skip data (relative to the list's first posting)
  uint64_t cand[kCand];
  uint2 wq[kThreads / 32][kWq];    // per-warp queues of (doc, tf word) awaiting their score / clause evaluation
  DevProbeQuery pq;                // the query's record, copied whole by every item (an item patches kind and row)
  uint64_t stage_bar;
  // per slot, of the item (CTA-uniform, written between the set-up barriers)
  uint32_t s_ia[kT], s_ib[kT];     // item bounds (postings relative to the list's first)
  uint32_t s_ra[kT], s_rb[kT];     // run bounds
  int32_t s_sdelta[kT];            // staged lists: smem index of posting x = x + s_sdelta
  uint32_t s_need[kT];             // slots a driver posting of this slot probes
  uint32_t s_candbelow[kT];        // word bytes of the lists that own a doc before this slot (candidate emission)
  uint32_t s_cntbefore[kT];        // ... (hit counting)
  uint32_t s_pre[kT + 1];          // prefix of the driver postings of the run
  uint32_t drv_mask, ess_mask, plane_mask, long_mask, short_mask, global_mask;
  int32_t short_total;             // staged postings of the short lists (aligned)
  int32_t g1;                      // end of the current run (granule of the slice)
  int32_t run_d0, run_d1;          // doc range of the current run
  int32_t staged;                  // the current run issued TMA copies
  int wi;
  int skip;                        // the claimed item is not processed (abort flag set)
  int cand_count;
  unsigned long long hits0;
  unsigned long long hits_known;   // max(hits0, docs known to match)
  int theta_dec;                   // 1: the item publishes (k-th key - 1) as threshold (sweep warm-up: its candidates are not output)
  unsigned long long theta;
  int dbg_theta0;                  // profiling instantiation: the item started without a threshold
  // pure disjunctions: a regular item of a query with an exact sweep warm-up
  int32_t warm_g;                  // the warm-up's end granule, relative to the slice
  uint32_t warm_own;               // the word byte of the warm-up's list: below warm_g, a doc that holds it is the warm-up's
  uint32_t s_candrun[kT], s_cntrun[kT];   // s_candbelow / s_cntbefore in the current run: with warm_own in a run below warm_g
  uint32_t run_drv;                // the lists that lead in the run (drv_mask without the warm-up's list below warm_g)
};
static_assert(sizeof(ProbeSmemT<kStageA>) <= 232448 / kCtasA - 1024 && sizeof(ProbeSmemT<kStageB>) <= 232448 / kCtasB - 1024, "ProbeSmem exceeds the per-CTA shared memory budget");

// A staged segment [a, b) of a list (postings relative to the list's first) is copied from the enclosing 16-posting
// aligned range of the GLOBAL posting arrays (TMA needs 16-byte aligned tf bytes): with pbm = post_base mod 16 the
// copy starts at list-relative posting seg_first(a, pbm) (may be negative: the tail of the previous list) and holds
// seg_n(a, b, pbm) postings.
__device__ __forceinline__ int32_t seg_first(uint32_t a, uint32_t pbm) { return (int32_t)((a + pbm) & ~(uint32_t)(kAlign - 1)) - (int32_t)pbm; }
__device__ __forceinline__ uint32_t seg_n(uint32_t a, uint32_t b, uint32_t pbm) {
  return b > a ? ((b + pbm + kAlign - 1) & ~(uint32_t)(kAlign - 1)) - ((a + pbm) & ~(uint32_t)(kAlign - 1)) : 0u;
}

// the clauses of sm.pq.q on one queued doc; word holds the doc's tf byte of every term slot (kTfInexact: a saturated 2-bit
// code, the exact byte is read from the byte plane). The norm byte is reused while consecutive scored
// term clauses read one field.
template <typename SM>
__device__ __noinline__ bool evaluate_doc(const ProbeLaunch& L, const SM& sm, int32_t doc, uint32_t word, float* out_score) {
  int cur_field = -1;
  uint32_t nb = 1u;
  auto term = [&](const DevClause& c, float* s) {
    uint32_t b = (word >> (8 * c.slot)) & 0xffu;
    if (b == 0) return false;
    if (c.scoring) {
      if (b == kTfInexact && sm.pq.plane[c.slot]) b = (uint32_t)__ldg(sm.pq.plane[c.slot] + doc);
      if (c.field != cur_field) {
        cur_field = c.field;
        const uint8_t* nrm = L.ix.norms[c.field];
        nb = nrm ? (uint32_t)__ldg(nrm + doc) : 1u;
      }
      const float f = (b == 255u) ? exact_freq_slow(L.ix, c, doc) : (float)b;
      *s = bm25_score(c.weight, f, __ldg(&L.ix.caches[c.field * 256 + nb]));
    }
    return true;
  };
  return eval_clauses(L.ix, sm.pq.q, sm.pq.cl, doc, presence4(word), term, out_score);
}

// exact score of a doc of a pure single-field disjunction: double sum, in slot (= clause) order, of Lucene's BM25 float
// expression for the slots present (BM25Scorer.score; DisjunctionSumScorer / MaxScoreBulkScorer sum in double)
template <typename SM>
__device__ __forceinline__ float score_disjunction(const ProbeLaunch& L, const SM& sm, const uint8_t* norms0, int n_term,
                                                   int32_t doc, uint32_t word) {
  const uint32_t nb = norms0 ? (uint32_t)__ldg(norms0 + doc) : 1u;
  double sum = 0.0;
#pragma unroll
  for (int s = 0; s < kT; ++s) {
    if (s >= n_term) break;
    uint32_t b = (word >> (8 * s)) & 0xffu;
    if (b == 0) continue;
    if (b == kTfInexact && sm.pq.plane[s]) b = (uint32_t)__ldg(sm.pq.plane[s] + doc);   // saturated 2-bit code: the exact byte
    const float f = (b == 255u) ? exact_freq_slow(L.ix, sm.pq.cl[sm.pq.clause[s]], doc) : (float)b;
    sum += (double)bm25_score(sm.pq.weight[s], f, __ldg(&L.ix.caches[sm.pq.field[s] * 256 + nb]));
  }
  return (float)sum;
}

// Candidate buffer flush (all threads; the buffer holds keys only): keeps the best top_k, publishes the k-th key (minus
// theta_dec) as the query's threshold.
template <typename SM>
__device__ __noinline__ void flush_candidates(const ProbeLaunch& L, SM& sm, int top_k, uint64_t* g_theta) {
  const long long ts = L.stats ? clock64() : 0ll;
  flush_top_k(sm.cand, sm.cand_count, kCand, top_k, (unsigned long long)sm.theta_dec, g_theta, sm.theta);
  if (L.stats && threadIdx.x == 0) atomicAdd(&L.stats[15], (unsigned long long)(clock64() - ts));
}

// binary search of doc in the sorted smem range [l, h); returns the tf byte (0 = absent)
template <typename SM>
__device__ __forceinline__ uint32_t probe_smem(const SM& sm, int l, int h, int32_t doc) {
  const int end = h;
  while (l < h) {
    const int mid = (l + h) >> 1;
    if (sm.sdocs[mid] < doc) l = mid + 1; else h = mid;
  }
  return (l < end && sm.sdocs[l] == doc) ? (uint32_t)sm.sf8[l] : 0u;
}
__device__ __noinline__ uint32_t probe_global(const int32_t* docs, const uint8_t* f8, uint32_t l, uint32_t h, int32_t doc) {
  const uint32_t end = h;
  while (l < h) {
    const uint32_t mid = (l + h) >> 1;
    if (__ldg(docs + mid) < doc) l = mid + 1; else h = mid;
  }
  return (l < end && __ldg(docs + l) == doc) ? (uint32_t)__ldg(f8 + l) : 0u;
}

// MAXSCORE split of a pure disjunction: the slots whose list-wide bounds sum (double, ascending) below theta.score are
// non-essential -- they never lead, docs found only in them cannot enter the top-k. Pruning needs a threshold and, in
// TOP_SCORES, more hits known than totalHitsThreshold (hits_known by reference: read only once theta is set).
__device__ __forceinline__ uint32_t maxscore_nonessential(const DevProbeQuery& pq, int n_term, unsigned long long theta, bool complete,
                                                          const unsigned long long& hits_known, int64_t threshold) {
  uint32_t ne = 0;
  if (theta != 0ull && (complete || (int64_t)hits_known > threshold)) {
    const float theta_s = key_score(theta);
    for (int a = 0; a < n_term; ++a) {
      if (!(pq.pre[a] < theta_s)) break;
      ne |= 1u << pq.ord[a];
    }
  }
  return ne;
}

// Profiling instantiation, end of a pure-disjunction item (thread 0): the MAXSCORE roles it swept with, against the split
// the query's threshold and hit count give now. A strict superset of non-essential lists marks an item that led with
// lists a later split would not have led with; their postings bound what refreshing the roles inside the item could save.
template <typename SM>
__device__ __noinline__ void count_role_stats(const ProbeLaunch& L, const SM& sm, int qi, int slice, uint32_t ess_mask,
                                              unsigned long long cyc, unsigned long long driver_postings) {
  const int n_term = sm.pq.q.n_term;
  const uint32_t all = (1u << n_term) - 1u;
  const bool complete = L.threshold >= (int64_t)INT32_MAX;
  const unsigned long long theta = *(volatile unsigned long long*)&L.theta[qi];
  const unsigned long long hits = *(volatile unsigned long long*)&L.total_hits[qi];
  const unsigned long long hits_known = hits > sm.hits_known ? hits : sm.hits_known;
  const uint32_t ne0 = all & ~ess_mask;
  const uint32_t ne1 = maxscore_nonessential(sm.pq, n_term, theta > sm.theta ? theta : sm.theta, complete, hits_known, L.threshold);
  if (sm.dbg_theta0) atomicAdd(&L.stats[19], cyc);
  if ((ne1 & ne0) == ne0 && ne1 != ne0) {
    unsigned long long turned = 0;   // postings of the item's lists that turned non-essential
    for (int s = 0; s < n_term; ++s) if (((ne1 & ~ne0) >> s) & 1u) turned += sm.s_ib[s] - sm.s_ia[s];
    atomicAdd(&L.stats[22], 1ull); atomicAdd(&L.stats[23], cyc); atomicAdd(&L.stats[24], driver_postings); atomicAdd(&L.stats[25], turned);
    if (slice <= 1) atomicAdd(&L.stats[26 + slice], 1ull);
  }
}

// kStats: the profiling instantiation (NRTGPU_DEBUG_MODES=1) keeps cycle counters; the production one has none of their registers
// kMulti: the generic instantiation for launches whose collectors count a SORTED_SET keyword column (agg_collect<true>)
template <bool kSimple, bool kStats, int kCtas, int kStageT, bool kMulti = false>
__global__ void __launch_bounds__(kThreads, kCtas) posting_probe_kernel(const __grid_constant__ ProbeLaunch L) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  using ProbeSmem = ProbeSmemT<kStageT>;
  constexpr int kStage = kStageT, kShortMax = ProbeSmem::kShortMax;
  ProbeSmem& sm = *reinterpret_cast<ProbeSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  if (tid == 0) {
    mbar_init(&sm.stage_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  uint32_t stage_parity = 0;   // phase of stage_bar the next staged run completes (tracked identically by every thread)
  const int gran_per_slice = L.slice_docs >> kLogGran;
  const int fine = (gran_per_slice + L.parts_max - 1) / L.parts_max;   // granules per finest part of a slice
  const int sb_stride = boundary_entries(L.n_slices, L.parts_max);
  const long long t_cta = kStats ? clock64() : 0ll;

  for (;;) {
    __syncthreads();   // the previous item is retired (also orders the mbarrier init before its first use)
    if (tid == 0) {
      const int w = (int)atomicAdd(L.work_counter, 1u);
      sm.wi = w;
      sm.skip = 0;
      if (L.deadline_ns && w < L.n_work && deadline_passed(L.deadline_ns, L.clock0)) {
        sm.skip = 1; L.timed_out[L.work_query[w]] = 1;   // drain the queue
      }
    }
    __syncthreads();
    const int wi = sm.wi;
    if (wi >= L.n_work) break;
    if (sm.skip) continue;
    const long long t_start = kStats ? clock64() : 0ll;
    const int qi = L.work_query[wi];
    const int32_t item = L.work_slice[wi];
    const int slice = item_slice(item);
    const int wflags = item_flags(item);
    // Sweep warm-up item (kItemSweep): the first 32K postings of the query's highest-bound list, over the WHOLE shard,
    // probing only the lists with tf planes (the other lists count as absent: scores are lower bounds). Nothing is output;
    // the k-th best lower-bound key minus one becomes the query's threshold before any other item of the query runs --
    // the docs that hold the query's rarest term are where its top-k is, a far better sample than the first 32K docs.
    // EXACT sweep warm-up (the record's warm_slot, TOP_SCORES, every other list has a plane): nothing is absent, so the
    // keys are true keys. It sweeps the list up to the record's warm_gran (the first granule boundary with 32K postings
    // below it), counts and outputs those docs like a regular item and publishes the k-th key; in the query's other items
    // the list leads only from warm_gran on, and below it a doc that holds the list is the warm-up's (run_drv, s_candrun,
    // s_cntrun).
    const bool sweep_warm = (wflags & kItemSweep) != 0;
    const int warm_slot = item_sweep_slot(item);
    const int g_first = slice * gran_per_slice;
    const int g_count = min(gran_per_slice, L.n_gran - g_first);
    // granule range of the item inside its slice, and the entries of the boundary table that hold its posting bounds
    const ItemSpan span = item_span(item, g_count, fine, L.parts_max, L.n_slices);
    const int g_lo = span.g_lo, g_hi = span.g_hi;
    // ---- everything that needs only the item word: the query's record (16 bytes per thread; ubt only where it is
    // read), the item's posting bounds, the query's threshold and hit count, and one step behind the record's rows the
    // granule offsets of the lists with skip data. Every load is issued before the first value is stored, so that the
    // set-up costs two dependent round trips and not one per loop iteration.
    {
      constexpr int n16 = (int)((kSimple ? sizeof(DevProbeQuery) : offsetof(DevProbeQuery, ubt)) / 16);
      static_assert(n16 <= kThreads && kThreads == 64 * kT, "one 16-byte piece per thread; 64 threads per slot's granule offsets");
      constexpr int kGbIter = (kMaxSliceGran + 1 + 63) / 64;
      const int gs = tid >> 6, gj = g_lo + (tid & 63);   // this thread's slot and first granule of gb[]
      const int gran_row = sweep_warm ? -1 : __ldg(&L.pquery[qi].row[gs]);
      uint4 piece = make_uint4(0u, 0u, 0u, 0u);
      if (tid < n16) piece = __ldg(reinterpret_cast<const uint4*>(L.pquery + qi) + tid);
      unsigned long long theta = 0ull, hits0 = 0ull, known = 0ull;
      uint32_t ba = 0, bb = 0, bw = 0, bx = 0;
      int exact_slot = -1;
      if (tid == 0) {
        theta = *(volatile unsigned long long*)&L.theta[qi];
        hits0 = *(volatile unsigned long long*)&L.total_hits[qi];
        if (L.known_hits) known = L.known_hits[qi];
      }
      if (tid >= 32 && tid < 32 + kT) {   // (the boundary entries of a slot without a term clause are 0)
        const uint32_t* sb = L.sbounds + ((size_t)qi * kT + (tid - 32)) * sb_stride;
        ba = sb[span.e_lo];
        bb = sb[span.e_hi];
        if (wflags & kItemBehindWarm) bw = sb[boundary_warm_entry(L.n_slices, L.parts_max)];
        if (kSimple && sweep_warm) { exact_slot = __ldg(&L.pquery[qi].warm_slot); bx = sb[boundary_exact_entry(L.n_slices, L.parts_max)]; }
      }
      uint32_t gv[kGbIter];
      const uint32_t* row = L.ix.gran_tab + (size_t)max(gran_row, 0) * (size_t)(L.n_gran + 1) + g_first;
#pragma unroll
      for (int k = 0; k < kGbIter; ++k) gv[k] = (gran_row >= 0 && gj + 64 * k <= g_hi) ? __ldg(row + gj + 64 * k) : 0u;
      if (tid < n16) reinterpret_cast<uint4*>(&sm.pq)[tid] = piece;
      if (tid == 0) {
        sm.cand_count = 0;
        sm.theta = theta; sm.hits0 = hits0; sm.hits_known = known > hits0 ? known : hits0;
        sm.theta_dec = sweep_warm ? 1 : 0;
      }
      if (tid >= 32 && tid < 32 + kT) {
        const int s = tid - 32;
        const uint32_t a = max(ba, bw);
        if (sweep_warm && s == warm_slot) bb = (s == exact_slot) ? bx : min(bb, a + kSweepPostings);
        sm.s_ia[s] = a; sm.s_ib[s] = max(a, bb); sm.s_ra[s] = 0; sm.s_rb[s] = 0; sm.s_sdelta[s] = 0;
      }
#pragma unroll
      for (int k = 0; k < kGbIter; ++k) if (gran_row >= 0 && gj + 64 * k <= g_hi) sm.gb[gs][gj + 64 * k] = gv[k];
    }
    __syncthreads();   // B1: record, item bounds, threshold, granule offsets
    // terminateAfter (TerminateAfterWrapper.java:150-162): a query that has collected enough hits stops collecting
    if (L.terminate_after > 0 && (long long)sm.hits0 >= L.terminate_after) {
      if (tid == 0) L.terminated[qi] = 1;
      continue;
    }
    const int n_term = sm.pq.q.n_term;
    // ---- roles: one thread per slot (each derives the CTA-uniform split for itself), then thread 0 plans the staging
    if (tid < kT) {
      const int t = tid;
      const uint32_t all = (n_term >= 32) ? 0xffffffffu : ((1u << n_term) - 1u);
      const bool complete = L.threshold >= (int64_t)INT32_MAX;
      const uint32_t ne = (kSimple && !sweep_warm) ? maxscore_nonessential(sm.pq, n_term, sm.theta, complete, sm.hits_known, L.threshold) : 0u;
      uint32_t pm = 0;
      for (int s = 0; s < n_term; ++s) if (sm.pq.kind[s] == kPlane) pm |= 1u << s;
      uint32_t drv, ess;
      int cnt_first = -1;
      const bool exact_warm = kSimple && sm.pq.warm_slot >= 0;   // the query has an exact sweep warm-up
      if (kSimple && sweep_warm) {
        drv = ess = 1u << warm_slot;
        // (cntbefore: a lower-bound warm-up counts nothing, an exact one every live doc)
        if (t < n_term) { sm.s_candbelow[t] = 0u; sm.s_cntbefore[t] = exact_warm ? 0u : 0xffffffffu; sm.s_need[t] = pm & ~(1u << t); }
      } else if (kSimple) {
        ess = all & ~ne;
        if (complete && ne && !L.ix.live_bits) {   // the densest non-essential list with a plane contributes its posting count unread
          uint32_t best = 0;
          for (int s = 0; s < n_term; ++s)
            if (((ne & pm) >> s) & 1u) { const uint32_t n = sm.s_ib[s] - sm.s_ia[s]; if (n >= best) { best = n; cnt_first = s; } }
        }
        drv = complete ? (cnt_first >= 0 ? all & ~(1u << cnt_first) : all) : ess;
        if (t < n_term) {
          const uint32_t lower = (1u << t) - 1u;   // the slots before t
          const uint32_t first = cnt_first >= 0 ? 1u << cnt_first : 0u;
          const uint32_t below_ess = expand4(ess & lower);
          const uint32_t before_cnt = expand4((lower | first) & ~(1u << t));
          sm.s_candbelow[t] = below_ess;
          sm.s_cntbefore[t] = complete ? before_cnt : below_ess;
          // a non-essential list is swept only to count: it probes the earlier lists (and the one counted unread)
          sm.s_need[t] = (complete && !((ess >> t) & 1u)) ? ((lower | first) & ~(1u << t)) : (all & ~(1u << t));
        }
      } else {
        ess = sm.pq.q.dense_driver ? 0u : (sm.pq.q.driver_mask & all);   // dense: every doc of the slice is visited, all lists are probed
        drv = ess;
        if (t < n_term) {
          const uint32_t below = expand4(drv & ((1u << t) - 1u));
          sm.s_candbelow[t] = below; sm.s_cntbefore[t] = below;
          sm.s_need[t] = all & ~(1u << t);
        }
      }
      // sweep warm-up: a list without a plane is not probed and counts as absent (scores are lower bounds), nothing is
      // narrowed by granule. The record's ubt still holds: a slot that is not probed has tf code 0 in every table index,
      // and the pattern sums of such indexes add (double)0 for it whatever its kind.
      __syncwarp((1u << kT) - 1u);   // every lane has read the record's kinds
      if (sweep_warm) {
        if (sm.pq.kind[t] != kPlane && t != warm_slot) sm.pq.kind[t] = kAbsent;
        sm.pq.row[t] = -1;
      }
      __syncwarp((1u << kT) - 1u);
      if (t == 0) {
        if (ne && !complete) L.pruned[qi] = 1;
        if (kSimple) {
          if (exact_warm && sweep_warm) sm.theta_dec = 0;
          const int warm_g = (exact_warm && !sweep_warm) ? sm.pq.warm_gran - g_first : 0;
          sm.warm_g = warm_g;
          sm.warm_own = exact_warm ? 0xffu << (8 * sm.pq.warm_slot) : 0u;
          if (exact_warm && !sweep_warm && warm_g >= g_hi) drv &= ~(1u << sm.pq.warm_slot);   // the warm-up swept the list's postings of the item
        }
        // short lists are staged whole at the first run; what does not fit the reserve is searched in global memory
        int st = 0;
        uint32_t lm = 0, shm = 0, gm = 0;
        for (int s = 0; s < n_term; ++s) {
          const int k = sm.pq.kind[s];
          if (k == kLong) lm |= 1u << s;
          else if (k == kShort) {
            const uint32_t a = sm.s_ia[s], b = sm.s_ib[s];
            const int need = (int)seg_n(a, b, sm.pq.pbm[s]);
            if (st + need <= kShortMax) { sm.s_sdelta[s] = st - seg_first(a, sm.pq.pbm[s]); st += need; shm |= 1u << s; }
            else { sm.pq.kind[s] = kGlobal; gm |= 1u << s; }
          }
        }
        if (sweep_warm) { st = 0; lm = 0; shm = 0; gm = 0; }   // the leading list is read in place, nothing is staged or searched
        sm.short_total = st;
        sm.plane_mask = pm; sm.long_mask = lm; sm.short_mask = shm; sm.global_mask = gm;
        if (cnt_first >= 0 && g_lo < g_hi)
          atomicAdd(&L.total_hits[qi], (unsigned long long)(sm.s_ib[cnt_first] - sm.s_ia[cnt_first]));
        sm.drv_mask = drv; sm.ess_mask = ess;
        if (kStats) {
          sm.dbg_theta0 = kSimple && !sweep_warm && sm.theta == 0ull;
          if (sm.dbg_theta0) { atomicAdd(&L.stats[18], 1ull); if (slice <= 1) atomicAdd(&L.stats[20 + slice], 1ull); }
        }
      }
    }
    __syncthreads();   // B2: roles, staging plan

    const int32_t slice_base = slice * L.slice_docs;
    const uint32_t drv_mask = sm.drv_mask, ess_mask = sm.ess_mask;
    const uint32_t plane_mask = sm.plane_mask, long_mask = sm.long_mask, short_mask = sm.short_mask, global_mask = sm.global_mask;
    unsigned int my_hits = 0;
    unsigned long long dbg_post = 0; unsigned int dbg_runs = 0, dbg_rounds = 0, dbg_flush = 0, dbg_staged = 0, dbg_queued = 0, dbg_admit = 0;
    long long dbg_tflush = 0, dbg_twait = 0;
    const long long t_setup = kStats ? clock64() : 0ll;

    const bool dense = !kSimple && sm.pq.q.dense_driver != 0;
    const uint32_t* live = L.ix.live_bits;
    const uint32_t sort_missing = (!kSimple && L.sort_kind == NRTGPU_SORT_COLUMN) ? *L.sort_missing_code : 0u;
    int g0 = g_lo;
    if (drv_mask == 0u && !dense) g0 = g_hi;   // nothing leads (every list non-essential): the slice cannot contribute
    bool first_run = true;
    while (g0 < g_hi) {
      // ---------------- run = the longest granule range [g0, g1) whose long-list segments fit the stage
      if (tid == 0) {
        { const unsigned long long g = *(volatile unsigned long long*)&L.theta[qi]; if (g > sm.theta) sm.theta = g; }
        const int cap = kStage - sm.short_total;
        auto fits = [&](int g1) {
          int tot = 0;
#pragma unroll
          for (int s = 0; s < kT; ++s)
            if ((long_mask >> s) & 1u) tot += (int)seg_n(sm.gb[s][g0], sm.gb[s][g1], sm.pq.pbm[s]);
          return tot <= cap;
        };
        int hi = g_hi, lo = g0 + 1;
        // no run straddles the end of an exact warm-up: below it, the warm-up's list does not lead (it is still staged and
        // probed) and a doc that holds it is owned by the warm-up
        // (the generic instantiation has no exact warm-ups: its items read s_candbelow, s_cntbefore and drv_mask)
        uint32_t run_drv = drv_mask;
        if (kSimple) {
          if (g0 < sm.warm_g && sm.warm_g < hi) hi = sm.warm_g;
          const uint32_t own = g0 < sm.warm_g ? sm.warm_own : 0u;
          for (int s = 0; s < kT; ++s) { sm.s_candrun[s] = sm.s_candbelow[s] | own; sm.s_cntrun[s] = sm.s_cntbefore[s] | own; }
          run_drv &= ~presence4(own);
          sm.run_drv = run_drv;
        }
        if (long_mask && hi > lo && !fits(hi)) {
          while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (fits(mid)) lo = mid; else hi = mid; }
          hi = lo;
        }
        const int g1 = hi;
        sm.g1 = g1;
        const bool whole = (g0 == g_lo && g1 == g_hi);
        const int32_t d0 = slice_base + (g0 << kLogGran);
        const int64_t d1_64 = (int64_t)slice_base + ((int64_t)g1 << kLogGran);
        const int32_t d1 = d1_64 > (int64_t)L.ix.n_docs ? L.ix.n_docs : (int32_t)d1_64;
        sm.run_d0 = d0; sm.run_d1 = d1;
        // run bounds of every list: skip data where the list has it, else a search by doc (staged short lists: in shared
        // memory once resident -- their first-run bounds are fixed up below; lists read from global memory: there)
        for (int s = 0; s < n_term; ++s) {
          const int k = sm.pq.kind[s];
          uint32_t a = sm.s_ia[s], b = sm.s_ib[s];
          if (sm.pq.row[s] >= 0) { a = max(a, sm.gb[s][g0]); b = min(b, sm.gb[s][g1]); }
          else if (!whole && b > a) {
            if (k == kShort) {
              if (!first_run) {
                const int base = sm.s_sdelta[s];
                int l = base + (int)a, h = base + (int)b;
                while (l < h) { const int m = (l + h) >> 1; if (sm.sdocs[m] < d0) l = m + 1; else h = m; }
                const uint32_t na = (uint32_t)(l - base);
                h = base + (int)b;
                while (l < h) { const int m = (l + h) >> 1; if (sm.sdocs[m] < d1) l = m + 1; else h = m; }
                a = na; b = (uint32_t)(l - base);
              }
            } else {   // kPlane without skip data, kGlobal
              const int32_t* gd = sm.pq.gdocs[s];
              uint32_t l = a, h = b;
              while (l < h) { const uint32_t m = (l + h) >> 1; if (__ldg(gd + m) < d0) l = m + 1; else h = m; }
              const uint32_t na = l;
              h = b;
              while (l < h) { const uint32_t m = (l + h) >> 1; if (__ldg(gd + m) < d1) l = m + 1; else h = m; }
              a = na; b = l;
            }
          }
          if (b < a) b = a;
          sm.s_ra[s] = a; sm.s_rb[s] = b;
        }
        // TMA copies: short lists once per item (first run, whole item segment), long lists per run behind them
        uint32_t total = 0;
        if (first_run)
          for (int s = 0; s < n_term; ++s)
            if ((short_mask >> s) & 1u) total += seg_n(sm.s_ia[s], sm.s_ib[s], sm.pq.pbm[s]) * 5u;
        for (int s = 0; s < n_term; ++s)
          if ((long_mask >> s) & 1u) total += seg_n(sm.s_ra[s], sm.s_rb[s], sm.pq.pbm[s]) * 5u;
        sm.staged = total != 0u;
        if (total) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy reads of the stage precede the async writes
          mbar_arrive_expect_tx(&sm.stage_bar, total);
          auto stage = [&](int s, uint32_t a, uint32_t b, int at) {   // copy the aligned range around [a, b) to sdocs/sf8[at...]
            const uint32_t pbm = sm.pq.pbm[s];
            const int32_t f = seg_first(a, pbm);
            const uint32_t n = seg_n(a, b, pbm);
            sm.s_sdelta[s] = at - f;
            const unsigned char* gd = reinterpret_cast<const unsigned char*>(sm.pq.gdocs[s] + f);
            const unsigned char* gf = reinterpret_cast<const unsigned char*>(sm.pq.gf8[s] + f);
            unsigned char* dd = reinterpret_cast<unsigned char*>(&sm.sdocs[at]);
            unsigned char* df = reinterpret_cast<unsigned char*>(&sm.sf8[at]);
            for (uint32_t o = 0; o < n * 4u; o += kPiece) bulk_g2s(dd + o, gd + o, min(kPiece, n * 4u - o), &sm.stage_bar);
            for (uint32_t o = 0; o < n; o += kPiece) bulk_g2s(df + o, gf + o, min(kPiece, n - o), &sm.stage_bar);
            return (int)n;
          };
          if (first_run)
            for (int s = 0; s < n_term; ++s)
              if (((short_mask >> s) & 1u) && sm.s_ib[s] > sm.s_ia[s])
                stage(s, sm.s_ia[s], sm.s_ib[s], sm.s_sdelta[s] + seg_first(sm.s_ia[s], sm.pq.pbm[s]));
          int st = sm.short_total;
          for (int s = 0; s < n_term; ++s)
            if (((long_mask >> s) & 1u) && sm.s_rb[s] > sm.s_ra[s]) st += stage(s, sm.s_ra[s], sm.s_rb[s], st);
        }
        uint32_t pre = 0;   // prefix of the driver postings
        for (int s = 0; s < kT; ++s) { sm.s_pre[s] = pre; if (s < n_term && ((run_drv >> s) & 1u)) pre += sm.s_rb[s] - sm.s_ra[s]; }
        sm.s_pre[kT] = pre;
      }
      __syncthreads();   // R1: run plan visible
      const int g1 = sm.g1;
      if (sm.staged) {
        const long long tw = kStats ? clock64() : 0ll;
        while (!mbar_try_wait(&sm.stage_bar, stage_parity)) {}
        stage_parity ^= 1u;
        if (kStats) dbg_twait += clock64() - tw;
      }
      if (first_run && g1 < g_hi && short_mask) {   // multi-run item: narrow the (now resident) short lists to the first run's docs
        __syncthreads();
        if (tid == 0) {
          const int32_t d0 = slice_base + (g0 << kLogGran);
          const int64_t d1_64 = (int64_t)slice_base + ((int64_t)g1 << kLogGran);
          const int32_t d1 = d1_64 > (int64_t)L.ix.n_docs ? L.ix.n_docs : (int32_t)d1_64;
          for (int s = 0; s < n_term; ++s)
            if (((short_mask >> s) & 1u) && sm.s_ib[s] > sm.s_ia[s]) {
              const int base = sm.s_sdelta[s];
              int l = base + (int)sm.s_ia[s], h = base + (int)sm.s_ib[s];
              while (l < h) { const int m = (l + h) >> 1; if (sm.sdocs[m] < d0) l = m + 1; else h = m; }
              const uint32_t na = (uint32_t)(l - base);
              h = base + (int)sm.s_ib[s];
              while (l < h) { const int m = (l + h) >> 1; if (sm.sdocs[m] < d1) l = m + 1; else h = m; }
              sm.s_ra[s] = na; sm.s_rb[s] = (uint32_t)(l - base);
            }
          uint32_t pre = 0;
          for (int s = 0; s < kT; ++s) { sm.s_pre[s] = pre; if (s < n_term && (((kSimple ? sm.run_drv : drv_mask) >> s) & 1u)) pre += sm.s_rb[s] - sm.s_ra[s]; }
          sm.s_pre[kT] = pre;
        }
        __syncthreads();
      }
      if (kStats) ++dbg_runs;
      // ---------------- rounds over the driver postings of the run
      const uint32_t n_total = sm.s_pre[kT];
      if (kStats && tid == 0) { dbg_post += n_total; dbg_staged += sm.staged ? 1u : 0u; }
      // No barrier between rounds: every warp streams through its postings on its own. A thread whose candidate does
      // not fit the buffer parks it and stops; the CTA meets at the barrier below, flushes once, and the loop resumes.
      // Driver lists are swept one after the other, so everything that depends on the leading list (what to probe,
      // where its postings live, who owns a doc) is loop invariant.
      int ct = 0;           // driver slot this thread is working on
      uint32_t cb = 0;      // first posting (of the slot's run segment) of the thread's next round
      uint64_t park = 0ull;   // this thread's key that did not fit the buffer
      bool parked = false;
      // Per-warp queue of the (doc, tf word) pairs that passed the cheap tests of the round: most driver postings fail
      // them, so scoring (pure disjunctions) or the clause evaluation (generic queries) would run with a handful of lanes.
      // The queue is drained 32 entries at a time; qn is warp-uniform.
      uint2* const wq = sm.wq[tid >> 5];
      int qn = 0;
      const uint32_t q_req = sm.pq.q.req_term_mask, q_not = sm.pq.q.not_term_mask;
      auto drain = [&](int n_take) -> bool {   // evaluates the last n_take (<= 32) queued pairs; true: a lane had to park its key
        __syncwarp();
        bool fail = false;
        const bool have = lane < n_take;
        const uint2 e = have ? wq[qn - n_take + lane] : make_uint2(0u, 0u);
        qn -= n_take;
        const int32_t d = (int32_t)e.x;
        uint64_t entry = 0ull;   // a real key is never 0: 0 fails the threshold test below
        if (kSimple) {
          if (have) {   // (the query's norms and after key are read here: registers are scarce across the rounds)
            const uint8_t* norms0 = sm.pq.q.single_field >= 0 ? L.ix.norms[sm.pq.q.single_field] : nullptr;
            entry = make_key(score_disjunction(L, sm, norms0, n_term, d, e.y), d);
          }
        } else {
          float score;
          if (have && evaluate_doc(L, sm, d, e.y, &score)) {
            ++my_hits;
            if (L.aggs) agg_collect<kMulti>(*L.aggs, L.ix, qi, d, score);   // additional collectors see every matching doc
            if (L.sort_kind == NRTGPU_SORT_RELEVANCE || L.sort_kind == kSortScoreRank) {
              entry = make_key(score, d);
              // [score, ...] order: ties by the order's rank, which takes the doc's place; ordered(-s) == ~ordered(s) for reverse
              if (L.sort_kind == kSortScoreRank) entry = make_key(L.sort_reverse ? -score : score, (int32_t)__ldg(L.sort_codes + d));
            } else {   // TopFieldCollector: the key is the doc's sort value (order-preserving code), ties by doc id
              uint32_t code = 0;
              if (L.sort_kind == NRTGPU_SORT_COLUMN) { code = __ldg(L.sort_codes + d); if (code == 0u) code = sort_missing; }
              entry = ((uint64_t)sort_hi(L.sort_kind, L.sort_reverse, code, d) << 32) | (uint32_t)(~(uint32_t)d);
            }
          }
        }
        // sm.theta never decreases within an item, so a key dropped here would not survive a flush either
        const unsigned long long th = sm.theta;
        if (entry > th && !(sm.pq.q.has_after && !(entry < sm.pq.q.after_key)) && !NRT_KNOCK(4)) {
          if (kStats) ++dbg_admit;
          const int p = atomicAdd(&sm.cand_count, 1);
          if (p < kCand) sm.cand[p] = entry;
          else { park = entry; parked = true; fail = true; }
        }
        __syncwarp();
        return fail;
      };
      for (;;) {
        bool full = false;
        if (parked) {
          const int p = atomicAdd(&sm.cand_count, 1);
          if (p < kCand) { sm.cand[p] = park; parked = false; } else full = true;
        }
        // the warp moves together (its queue operations are collective); a queue left >= 32 by a full buffer is brought
        // below 32 before the sweep pushes again
        full = __any_sync(0xffffffffu, full);
        while (!full && qn >= 32) full = __any_sync(0xffffffffu, drain(32));
        const int ct_end = NRT_KNOCK(8) ? 0 : (dense ? n_term + 1 : n_term);   // dense: one more "list" = every doc of the run
        while (!full && ct < ct_end) {
          const bool t_dense = ct == n_term;
          const uint32_t n_t = t_dense ? (uint32_t)(sm.run_d1 - sm.run_d0) : ((((kSimple ? sm.run_drv : drv_mask) >> ct) & 1u) ? sm.s_rb[ct] - sm.s_ra[ct] : 0u);
          if (cb >= n_t) { ++ct; cb = 0; continue; }
          const int t = t_dense ? 0 : ct;
          const uint32_t need = t_dense ? ((n_term >= 32) ? 0xffffffffu : ((1u << n_term) - 1u)) : sm.s_need[t];
          const bool t_staged = !t_dense && (((long_mask | short_mask) >> t) & 1u);
          const bool t_ess = (ess_mask >> t) & 1u;
          const uint32_t candbelow = t_dense ? 0u : (kSimple ? sm.s_candrun[t] : sm.s_candbelow[t]),
                         cntbefore = t_dense ? 0u : (kSimple ? sm.s_cntrun[t] : sm.s_cntbefore[t]);
          const int32_t dense_d0 = sm.run_d0;
          const uint32_t tshift = t_dense ? 0u : 8u * (uint32_t)t;
          constexpr uint32_t kRound = kR * kThreads;
          constexpr int kP = kT - 1;   // slots a driver posting of a pure disjunction probes (every slot but its own)
          int32_t doc[kR], nd[kR]; uint32_t df[kR], nf[kR];
          uint32_t gq[kR][kP];         // (simple) the plane bytes of round r, gathered one round ahead
          // The simple instantiations read the driver list in one of two forms, fixed for all its rounds: staged (posting
          // x of the run segment at sdocs / sf8[sbase + x]) or in place (gdoc / gf8[x], read-only global loads).
          const int sbase = (int)sm.s_ra[t] + sm.s_sdelta[t];
          const int32_t* gdoc = sm.pq.gdocs[t] + sm.s_ra[t];
          const uint8_t* gf8 = sm.pq.gf8[t] + sm.s_ra[t];
          // The probe plan of a pure disjunction's driver list, built once per driver list and kept in registers for all
          // its rounds (the rounds store to shared memory, so the compiler would otherwise reload it per posting):
          // entries [0, np) are the slots gathered from a tf plane, pw = the plane's 2-bit codes; entries [np, n_probe)
          // the slots searched, pw = posting range a | b << 32 with pd = the shared-memory index of posting 0 (long: a
          // granule of [a, b) is searched; short: the whole range; global: [a, b) of the list in global memory). Byte i
          // of pslot: the slot of entry i and, for a search, its kind << 2. A search of an empty range finds nothing, so
          // such a slot is left out.
          uint64_t pw[kP]; int32_t pd[kP];
          uint32_t pslot = 0u;
          int np = 0, n_probe = 0;
          // postings of the round that starts at b0 (doc -1: no posting)
          auto fetch = [&](uint32_t b0, int32_t (&d)[kR], uint32_t (&f)[kR]) {
#pragma unroll
            for (int j = 0; j < kR; ++j) {
              const uint32_t x = b0 + (uint32_t)(j * kThreads + tid);
              d[j] = -1; f[j] = 0u;
              if (x < n_t) {
                if (t_staged) { d[j] = sm.sdocs[sbase + (int)x]; f[j] = sm.sf8[sbase + (int)x]; }
                else { d[j] = __ldg(gdoc + x); f[j] = __ldg(gf8 + x); }
              }
            }
          };
          // plane gathers of the postings of a round (2-bit tf codes, all in flight together; lanes without a posting
          // gather byte 0 of the plane: harmless, and the branches stay warp-uniform)
          auto gather = [&](const int32_t (&d)[kR], uint32_t (&g)[kR][kP]) {
#pragma unroll
            for (int j = 0; j < kR; ++j) {
              const uint32_t d4 = (uint32_t)max(d[j], 0) >> 2;
#pragma unroll
              for (int i = 0; i < kP; ++i) g[j][i] = i < np ? (uint32_t)__ldg(reinterpret_cast<const uint8_t*>(pw[i]) + d4) : 0u;
            }
          };
          // The generic instantiations keep the mask-driven round: what each slot is probed by, tested per posting, one
          // generic load path for staged (shared memory) and in-place (global memory) driver lists, postings one round
          // ahead and the round's gathers issued as it starts. With the plan they ran slower (DESIGN.md §4.1 Rounds):
          // their drains call the clause evaluation with every live register saved around the call.
          const uint32_t need_plane = NRT_KNOCK(1) ? 0u : need & plane_mask, need_long = NRT_KNOCK(2) ? 0u : need & long_mask,
                         need_short = NRT_KNOCK(2) ? 0u : need & short_mask, need_glob = need & global_mask;
          const int32_t* dptr = t_staged ? sm.sdocs + sbase : gdoc;
          const uint8_t* fptr = t_staged ? sm.sf8 + sbase : gf8;
          if constexpr (kSimple) {
            uint32_t rest_p = NRT_KNOCK(1) ? 0u : need & plane_mask;
            uint32_t rest_s = (NRT_KNOCK(2) ? 0u : need & (long_mask | short_mask)) | (need & global_mask);
            for (int u = 0; u < kT; ++u) if (((rest_s >> u) & 1u) && sm.s_rb[u] <= sm.s_ra[u]) rest_s &= ~(1u << u);
            np = __popc(rest_p);
            n_probe = np + __popc(rest_s);
#pragma unroll
            for (int i = 0; i < kP; ++i) {
              pw[i] = 0ull; pd[i] = 0;
              if (rest_p) {
                const int u = __ffs(rest_p) - 1;
                rest_p &= rest_p - 1u;
                pw[i] = reinterpret_cast<uint64_t>(sm.pq.plane2[u]);
                pslot |= (uint32_t)u << (8 * i);
              } else if (rest_s) {
                const int u = __ffs(rest_s) - 1;
                rest_s &= rest_s - 1u;
                const uint32_t kind = ((long_mask >> u) & 1u) ? kLong : (((short_mask >> u) & 1u) ? kShort : kGlobal);
                pw[i] = (uint64_t)sm.s_ra[u] | ((uint64_t)sm.s_rb[u] << 32);
                pd[i] = sm.s_sdelta[u];
                pslot |= ((uint32_t)u | (kind << 2)) << (8 * i);
              }
            }
            // Software pipeline, restarted from cb for every driver list and after every flush (nothing of it outlives a
            // round that did not complete): the postings of round r + 2 are fetched and the plane gathers of round r + 1
            // issued before round r is searched, tested and queued, so the gathers of a warp overlap its own searches.
            fetch(cb, doc, df);
            gather(doc, gq);
            fetch(cb + kRound, nd, nf);
          } else {
            np = need_plane != 0u;
#pragma unroll
            for (int j = 0; j < kR; ++j) {
              const uint32_t x = cb + (uint32_t)(j * kThreads + tid);
              nd[j] = -1; nf[j] = 0;   // doc -1: no posting
              if (x < n_t) {
                if (t_dense) nd[j] = dense_d0 + (int32_t)x; else { nd[j] = dptr[x]; nf[j] = fptr[x]; }
              }
            }
          }
          while (!full && cb < n_t) {
            const unsigned long long theta = sm.theta;
            const float theta_s = theta ? key_score(theta) : -INFINITY;
            uint32_t word[kR];
            uint32_t pbyte[kR][kT];   // (generic) the plane bytes of the round, by slot
            uint32_t ngq[kR][kP]; int32_t nnd[kR]; uint32_t nnf[kR];   // (simple) the next stages of the pipeline
            if constexpr (kSimple) {
              if (cb + kRound < n_t) gather(nd, ngq);
              else {
#pragma unroll
                for (int j = 0; j < kR; ++j)
#pragma unroll
                  for (int i = 0; i < kP; ++i) ngq[j][i] = 0u;
              }
              fetch(cb + 2 * kRound, nnd, nnf);
#pragma unroll
              for (int j = 0; j < kR; ++j) word[j] = df[j] << tshift;
              // searches (staged lists in shared memory)
              if (n_probe > np) {
#pragma unroll
                for (int j = 0; j < kR; ++j) {
                  if (doc[j] < 0) continue;
                  const int g = (doc[j] - slice_base) >> kLogGran;
#pragma unroll
                  for (int i = 0; i < kP; ++i) {
                    if (i < np || i >= n_probe) continue;
                    const uint32_t u = (pslot >> (8 * i)) & 3u, kind = (pslot >> (8 * i + 2)) & 7u;
                    const uint32_t a = (uint32_t)pw[i], b = (uint32_t)(pw[i] >> 32);
                    uint32_t r = 0;
                    if (kind == kLong) {
                      const uint32_t lo = max(sm.gb[u][g], a), hi = min(sm.gb[u][g + 1], b);
                      if (hi > lo) r = probe_smem(sm, (int)lo + pd[i], (int)hi + pd[i], doc[j]);
                    } else if (kind == kShort) {
                      r = probe_smem(sm, (int)a + pd[i], (int)b + pd[i], doc[j]);
                    } else {
                      r = probe_global(sm.pq.gdocs[u], sm.pq.gf8[u], a, b, doc[j]);
                    }
                    word[j] |= r << (8 * u);
                  }
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < kR; ++j) { doc[j] = nd[j]; word[j] = nf[j] << tshift; }
              // plane gathers of every posting of the round (2-bit tf codes, all in flight together)
              // (lanes without a posting gather byte 0 of the plane: harmless, and the branches stay CTA-uniform)
#pragma unroll
              for (int j = 0; j < kR; ++j) {
                const uint32_t d4 = (uint32_t)max(doc[j], 0) >> 2;
                pbyte[j][0] = 0u; pbyte[j][1] = 0u; pbyte[j][2] = 0u; pbyte[j][3] = 0u;
                if (need_plane & 1u) pbyte[j][0] = (uint32_t)__ldg(sm.pq.plane2[0] + d4);
                if (need_plane & 2u) pbyte[j][1] = (uint32_t)__ldg(sm.pq.plane2[1] + d4);
                if (need_plane & 4u) pbyte[j][2] = (uint32_t)__ldg(sm.pq.plane2[2] + d4);
                if (need_plane & 8u) pbyte[j][3] = (uint32_t)__ldg(sm.pq.plane2[3] + d4);
              }
              // next round's postings
              {
                const uint32_t nb = cb + kRound;
#pragma unroll
                for (int j = 0; j < kR; ++j) {
                  const uint32_t x = nb + (uint32_t)(j * kThreads + tid);
                  nd[j] = -1; nf[j] = 0;
                  if (x < n_t) {
                    if (t_dense) nd[j] = dense_d0 + (int32_t)x; else { nd[j] = dptr[x]; nf[j] = fptr[x]; }
                  }
                }
              }
              // searches of the staged lists (shared memory; overlaps the gathers)
              if (need_long | need_short | need_glob) {
#pragma unroll
                for (int j = 0; j < kR; ++j) {
                  if (doc[j] < 0) continue;
                  const int g = (doc[j] - slice_base) >> kLogGran;
#pragma unroll
                  for (int u = 0; u < kT; ++u) {
                    uint32_t b = 0;
                    if ((need_long >> u) & 1u) {
                      const uint32_t lo = max(sm.gb[u][g], sm.s_ra[u]), hi = min(sm.gb[u][g + 1], sm.s_rb[u]);
                      if (hi > lo) b = probe_smem(sm, (int)lo + sm.s_sdelta[u], (int)hi + sm.s_sdelta[u], doc[j]);
                    } else if ((need_short >> u) & 1u) {
                      if (sm.s_rb[u] > sm.s_ra[u]) b = probe_smem(sm, (int)sm.s_ra[u] + sm.s_sdelta[u], (int)sm.s_rb[u] + sm.s_sdelta[u], doc[j]);
                    } else if ((need_glob >> u) & 1u) {
                      if (sm.s_rb[u] > sm.s_ra[u]) b = probe_global(sm.pq.gdocs[u], sm.pq.gf8[u], sm.s_ra[u], sm.s_rb[u], doc[j]);
                    }
                    word[j] |= b << (8 * u);
                  }
                }
              }
            }
            // ownership, hit count and the cheap tests of every posting of the round, then the survivors are queued (the
            // gathered bytes are dead before the first drain)
            uint32_t surv_mask = 0;
#pragma unroll
            for (int j = 0; j < kR; ++j) {
              uint32_t v = word[j];
              if (np) {
                // the gathered bytes side by side; the doc's 2-bit code of every plane with one shift and one mask
                // (bits shifted in from the neighbouring byte fall outside the mask); code 3 = "three or more" becomes
                // kTfInexact (resolved when the doc is scored)
                uint32_t raw = 0u;
                if constexpr (kSimple) {
#pragma unroll
                  for (int i = 0; i < kP; ++i) raw |= gq[j][i] << (8u * ((pslot >> (8 * i)) & 3u));
                } else {
                  raw = pbyte[j][0] | (pbyte[j][1] << 8) | (pbyte[j][2] << 16) | (pbyte[j][3] << 24);
                }
                const uint32_t codes = (raw >> (((uint32_t)max(doc[j], 0) & 3u) * 2u)) & 0x03030303u;
                const uint32_t sat = __vcmpeq4(codes, 0x03030303u);   // 0xff where the code saturated
                v |= (codes & ~sat) | (sat & (kTfInexact * 0x01010101u));
              }
              bool surv = false;
              if (kSimple) {
                // deleted docs are neither counted nor collected; a doc owned by a lower list is counted there; a doc whose
                // tf-pattern bound is below the threshold cannot reach the top-k
                if (doc[j] >= 0 && !(live && !((live[doc[j] >> 5] >> (doc[j] & 31)) & 1u))) {
                  if ((v & cntbefore) == 0u) ++my_hits;
                  surv = t_ess && (v & candbelow) == 0u && !(sm.pq.ubt[__dp4a(__vminu4(v, 0x03030303u), 0x40100401u, 0u)] < theta_s);
                }
              } else {   // not owned by a lower list, every required term present, no excluded term
                const uint32_t pres = presence4(v);
                surv = doc[j] >= 0 && (v & candbelow) == 0u && (pres & q_req) == q_req && (pres & q_not) == 0u;
              }
              word[j] = v;
              surv_mask |= surv ? 1u << j : 0u;
            }
#pragma unroll
            for (int j = 0; j < kR; ++j) {
              const bool surv = (surv_mask >> j) & 1u;
              const unsigned bal = __ballot_sync(0xffffffffu, surv);
              if (surv) wq[qn + __popc(bal & ((1u << lane) - 1u))] = make_uint2((uint32_t)doc[j], word[j]);
              qn += __popc(bal);
              if (kStats && lane == 0) dbg_queued += __popc(bal);
              while (!full && qn >= 32) full = __any_sync(0xffffffffu, drain(32));   // (a parked key stops the warp: park is free whenever drain runs)
            }
            if constexpr (kSimple) {
#pragma unroll
              for (int j = 0; j < kR; ++j) {
                doc[j] = nd[j]; df[j] = nf[j]; nd[j] = nnd[j]; nf[j] = nnf[j];
#pragma unroll
                for (int i = 0; i < kP; ++i) gq[j][i] = ngq[j][i];
              }
            }
            cb += kRound;
            if (kStats && tid == 0) ++dbg_rounds;
          }
        }
        // the rest of the warp's queue (a partial warp), unless the buffer is full: then after the flush
        while (!full && qn > 0) full = __any_sync(0xffffffffu, drain(min(qn, 32)));
        __syncthreads();
        if (sm.cand_count <= kCand) break;   // nobody is parked (the count passes kCand only through a failed append)
        const long long tf = kStats ? clock64() : 0ll;
        flush_candidates(L, sm, L.top_k, &L.theta[qi]);
        if (kStats) dbg_tflush += clock64() - tf;
        if (kStats) ++dbg_flush;
      }
      g0 = g1;
      first_run = false;
      __syncthreads();   // R0: every thread is done with the stage before the next run overwrites it
    }

    // ---------------- finish the work item (the slice merge sorts, so only a full buffer needs ordering here)
    __syncthreads();
    if (sm.cand_count > L.top_k) {
      const long long tf = kStats ? clock64() : 0ll;
      flush_candidates(L, sm, L.top_k, &L.theta[qi]);
      if (kStats) dbg_tflush += clock64() - tf;
      if (kStats) ++dbg_flush;
    }
    const bool lb_warm = kSimple ? sm.theta_dec != 0 : sweep_warm;   // a lower-bound sweep warm-up outputs nothing and counts nothing
    const int keep = lb_warm ? 0 : min(sm.cand_count, L.top_k);
    const int out_list = item_out_list(item, L.parts_max, L.n_lists);
    uint64_t* out = L.slice_keys + ((size_t)qi * L.n_lists + out_list) * L.top_k;
    for (int i = tid; i < keep; i += kThreads) out[i] = sm.cand[i];
    if (tid == 0) L.slice_cnt[(size_t)qi * L.n_lists + out_list] = keep;
    for (int o = 16; o > 0; o >>= 1) my_hits += __shfl_xor_sync(0xffffffffu, my_hits, o);
    if (lane == 0 && my_hits && !lb_warm) atomicAdd(&L.total_hits[qi], (unsigned long long)my_hits);
    if (kStats) {
      for (int o = 16; o > 0; o >>= 1) dbg_admit += __shfl_xor_sync(0xffffffffu, dbg_admit, o);
      if (lane == 0) { atomicAdd(&L.stats[16], (unsigned long long)dbg_queued); atomicAdd(&L.stats[17], (unsigned long long)dbg_admit); }
    }
    if (kStats && tid == 0) {
      const unsigned long long cyc = (unsigned long long)(clock64() - t_start);
      atomicAdd(&L.stats[0], 1ull);
      atomicAdd(&L.stats[1], cyc);
      atomicAdd(&L.stats[2], (unsigned long long)dbg_runs);
      atomicAdd(&L.stats[3], dbg_post);
      atomicAdd(&L.stats[4], (unsigned long long)dbg_flush);
      atomicAdd(&L.stats[5], (unsigned long long)dbg_staged);
      atomicAdd(&L.stats[6], (unsigned long long)(t_setup - t_start));
      atomicAdd(&L.stats[7], (unsigned long long)dbg_rounds);
      atomicMax(&L.stats[8], cyc);
      if (wflags & (kItemWarmDocs | kItemSweep)) { atomicAdd(&L.stats[11], 1ull); atomicAdd(&L.stats[12], cyc); }
      if (sweep_warm && !lb_warm) { atomicAdd(&L.stats[28], 1ull); atomicAdd(&L.stats[29], dbg_post); atomicAdd(&L.stats[30], cyc); }
      atomicAdd(&L.stats[13], (unsigned long long)dbg_tflush); atomicAdd(&L.stats[14], (unsigned long long)dbg_twait);
      if (kSimple && !sweep_warm) count_role_stats(L, sm, qi, item_slice(item), ess_mask, cyc, dbg_post);
    }
  }
  if (kStats && tid == 0) {
    const unsigned long long busy = (unsigned long long)(clock64() - t_cta);
    atomicAdd(&L.stats[9], busy); atomicMax(&L.stats[10], busy);
  }
}

// postings of every (query, term slot) below each part boundary of every slice (parts_max equal granule ranges per
// slice), below the end of the shard, below the warm-up boundary of slice 0 and below the end of the query's exact sweep
// warm-up (its record's warm_gran: probe_query_kernel runs first)
struct SliceBoundsLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  const DevProbeQuery* pquery;
  int32_t nq, n_slices, slice_gran, n_gran, parts_max;
  uint32_t* sbounds;   // [nq][kT][boundary_entries]
};

__global__ void slice_bounds_kernel(SliceBoundsLaunch B) {
  const int per_slot = boundary_entries(B.n_slices, B.parts_max);
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B.nq * kT * per_slot) return;
  const int q = (int)(i / (kT * per_slot)), s = (int)((i / per_slot) % kT), e = (int)(i % per_slot);
  const DevQuery dq = B.queries[q];
  const int64_t gran = e == boundary_exact_entry(B.n_slices, B.parts_max) ? (int64_t)B.pquery[q].warm_gran
                                                                           : boundary_gran(e, B.n_slices, B.parts_max, B.slice_gran, B.n_gran);
  uint32_t out = 0;
  for (int c = 0; c < dq.n_clauses; ++c) {
    const DevClause cl = B.clauses[dq.clause_begin + c];
    if (cl.kind != NRTGPU_TERM || cl.slot != s) continue;
    if (cl.gran_row >= 0) { out = __ldg(B.ix.gran_tab + (size_t)cl.gran_row * (size_t)(B.n_gran + 1) + gran); break; }
    const int64_t target64 = gran << kLogGran;
    const int32_t target = target64 > (int64_t)B.ix.n_docs ? B.ix.n_docs : (int32_t)target64;
    const int32_t* docs = B.ix.post_docs + cl.post_base;
    int lo = 0, hi = cl.n_post;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(docs + mid) < target) lo = mid + 1; else hi = mid; }
    out = (uint32_t)lo;
    break;
  }
  B.sbounds[i] = out;
}

// the per-query records of a probe batch (DevProbeQuery, batch_plan.h): one CTA per query, once per prepared batch
struct ProbeQueryLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  const uint8_t* field_min_norm;
  const int32_t* warm_exact;   // [nq] the slot of the query's exact sweep warm-up, -1: none (WorkPlan::warm_exact)
  int32_t n_gran;
  DevProbeQuery* out;   // [nq]
};

__global__ void __launch_bounds__(kUbt) probe_query_kernel(ProbeQueryLaunch B) {
  __shared__ DevProbeQuery r;
  __shared__ float uval[kT][2];   // per-slot score bounds at tf = 1, 2 (shortest field length present)
  const int qi = blockIdx.x, tid = threadIdx.x;
  const DevQuery dq = B.queries[qi];
  const int ncl = dq.n_clauses, n_term = dq.n_term;
  if (tid == 0) r.q = dq;
  if (tid < kMaxClauses) r.cl[tid] = tid < ncl ? B.clauses[dq.clause_begin + tid] : DevClause{};
  if (tid >= 32 && tid < 32 + kT) {
    const int s = tid - 32;
    r.kind[s] = kAbsent; r.plane[s] = nullptr; r.plane2[s] = nullptr; r.gdocs[s] = nullptr; r.gf8[s] = nullptr;
    r.weight[s] = 0.f; r.ub[s] = 0.f; r.clause[s] = 0; r.field[s] = 0; r.pbm[s] = 0; r.row[s] = -1; r.ord[s] = 0; r.pre[s] = 0.f;
  }
  if (tid == 0) { r.warm_slot = -1; r.warm_gran = 0; r.reserved[0] = r.reserved[1] = 0; }
  __syncthreads();
  if (tid < ncl && r.cl[tid].kind == NRTGPU_TERM) {   // per-slot descriptors (one thread per clause)
    const DevClause& c = r.cl[tid];
    const int s = c.slot;
    r.gdocs[s] = B.ix.post_docs + c.post_base;
    r.gf8[s] = B.ix.post_f8 + c.post_base;
    const bool has_plane = c.plane >= 0 && B.ix.dense_tf != nullptr && B.ix.dense_tf2 != nullptr;
    r.plane[s] = has_plane ? B.ix.dense_tf + (size_t)c.plane * (size_t)B.ix.dense_stride : nullptr;
    r.plane2[s] = has_plane ? B.ix.dense_tf2 + (size_t)c.plane * (size_t)(B.ix.dense_stride >> 2) : nullptr;
    r.kind[s] = has_plane ? kPlane : (c.gran_row >= 0 ? kLong : kShort);
    r.weight[s] = c.weight; r.ub[s] = c.ub; r.clause[s] = tid; r.field[s] = c.field;
    r.pbm[s] = (uint32_t)(c.post_base & (int64_t)(kAlign - 1)); r.row[s] = c.gran_row;
  }
  if (tid >= 64 && tid < 64 + 2 * kT) {
    const int s = (tid - 64) >> 1, c = ((tid - 64) & 1) + 1;
    float u = 0.0f;
    for (int i = 0; i < ncl; ++i)
      if (r.cl[i].kind == NRTGPU_TERM && r.cl[i].slot == s) {
        const uint32_t nbmin = (dq.single_field >= 0 && B.field_min_norm) ? (uint32_t)B.field_min_norm[dq.single_field] : 0u;
        u = bm25_score(r.cl[i].weight, (float)c, __ldg(&B.ix.caches[r.cl[i].field * 256 + nbmin]));
      }
    uval[s][c - 1] = u;
  }
  __syncthreads();
  {
    // ubt[sum min(tf_s, 3) * 4^s]: the double clause sum with every term at the shortest field length present
    // (tf >= 3 bounded by the clause weight, the limit tf -> inf) -- an upper bound of the doc's score
    const int i = tid;
    const int c[kT] = {i & 3, (i >> 2) & 3, (i >> 4) & 3, i >> 6};
    double sum = 0.0;
#pragma unroll
    for (int t = 0; t < kT; ++t) {
      float u = 0.0f;
      if (r.kind[t] != kAbsent && c[t] > 0) u = (c[t] <= 2) ? uval[t][c[t] - 1] : r.weight[t];
      sum += (double)u;
    }
    r.ubt[i] = (float)sum;
  }
  if (tid == 0) {   // MAXSCORE order: insertion sort by ub (equal bounds keep slot order), running double sums
    int ord[kT]; int n = 0;
    for (int s = 0; s < n_term; ++s) ord[n++] = s;
    for (int a = 1; a < n; ++a) { const int x = ord[a]; int b = a - 1; while (b >= 0 && r.ub[ord[b]] > r.ub[x]) { ord[b + 1] = ord[b]; --b; } ord[b + 1] = x; }
    double pre = 0.0;
    for (int a = 0; a < n; ++a) { pre += (double)r.ub[ord[a]]; r.ord[a] = ord[a]; r.pre[a] = (float)pre; }
    // exact sweep warm-up: every other slot is probed through a plane; it ends at the first granule boundary with
    // kSweepPostings postings of its list below it (the shard end for a shorter list or one without granule offsets)
    int w = B.warm_exact[qi];
    for (int s = 0; s < n_term; ++s) if (w >= 0 && s != w && r.kind[s] != kPlane) w = -1;
    if (w >= 0) {
      int lo = 0, hi = B.n_gran;
      if (r.row[w] >= 0) {
        const uint32_t* row = B.ix.gran_tab + (size_t)r.row[w] * (size_t)(B.n_gran + 1);
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(row + mid) < kSweepPostings) lo = mid + 1; else hi = mid; }
      }
      r.warm_slot = w; r.warm_gran = hi;
    }
  }
  __syncthreads();
  const uint4* src = reinterpret_cast<const uint4*>(&r);
  uint4* dst = reinterpret_cast<uint4*>(B.out + qi);
  for (int i = tid; i < (int)(sizeof(DevProbeQuery) / 16); i += kUbt) dst[i] = src[i];
}

}  // namespace v3
}  // namespace nrtgpu
